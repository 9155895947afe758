/*
 * maxi_oracle.c -- TEST INFRASTRUCTURE ONLY. CPU restatement ("port") of the reference's
 * per-sample DSP hot path in plain C, behind oracle_api.h.
 *
 * Parity status: PINNED. tests/test_oracle_vs_reference.py compares every function below
 * bit-for-bit (fp64 and fp32 alike, integer state exactly) with the unmodified reference
 * compiled from /root/reference (oracle/_ref/libmaxiref.so), and tests/test_golden.py
 * compares it with the fixtures under tests/golden/ that were generated from that same
 * compiled reference by tests/golden/make_golden.py. The reference's own tests hold no
 * numeric expectations for this path (SURVEY.md section 4), so the compiled reference
 * is the only pin there is.
 *
 * Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference
 * legs may load this library; the product (maximilian_b200/) never does.
 *
 * Every function cites the reference lines it restates (paths relative to /root/reference).
 * Build with -ffp-contract=off: the reference's evaluation order, without fused
 * multiply-adds, is part of the contract (float FFT differs by 4e-6 of frame max otherwise).
 * Uninitialised reference members (maxiDelayline::phase, all of maxiEnv, maxiOsc::output,
 * mel filter column 0) are defined as zero, the value they have in zero-filled storage.
 */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#include "oracle_api.h"

/* src/maximilian.h:55-58 */
#define MAXI_PI 3.1415926535897932384626433832795
#define MAXI_TWOPI 6.283185307179586476925286766559
/* src/libs/fft.h:36-38 (glibc's M_PI has the same value) */
#define FFT_M_PI 3.14159265358979323846

const char* mxo_kind(void) { return "port"; }

/* ================================================================= voices */

typedef struct {
    mxo_chain chain;
    int V;
    double* p[MXO_P_COUNT]; /* parameter arrays, index = MXO_P_* */
    /* oscillator state: src/maximilian.h:172-177 (phase, output) */
    double* osc_out;        /* maxiOsc::output, read by square()/pulse() when no branch fires */
    /* filter state */
    double *f0, *f1, *f2;   /* lores/hires x,y | svf v0z,v1,v2 | biquad v[1],v[2] */
    double *cf[5];          /* svf g1,g2,g3,g4,k | biquad a0,a1,a2,b1,b2 */
    /* maxiEnv state: src/maximilian.h:895-917 */
    double *env_amp, *env_output;
    int64_t* env_holdcount;
    int32_t* env_flags;     /* attack | decay<<1 | sustain<<2 | hold<<3 | release<<4 */
    /* maxiDelayline state: src/maximilian.h:269,273 */
    int32_t* dl_phase;
    double* ring;           /* [V][delay_capacity] */
} bank_t;

static double* dalloc(size_t n, double fill) {
    double* a = (double*)malloc(sizeof(double) * (n ? n : 1));
    if (a) for (size_t i = 0; i < n; ++i) a[i] = fill;
    return a;
}

/* maxiSVF::setParams, src/maximilian.h:1322-1334 (sampleRate is a size_t there) */
static void svf_set_params(const bank_t* b, int v) {
    const double sr = (double)(size_t)b->chain.sample_rate;
    const double freq = b->p[MXO_P_CUTOFF][v], res = b->p[MXO_P_RESONANCE][v];
    const double g = tan(MAXI_PI * freq / sr);
    const double damping = res == 0 ? 0 : 1.0 / res;
    const double k = damping;
    const double ginv = g / (1.0 + g * (g + k));
    b->cf[0][v] = ginv;                    /* g1 */
    b->cf[1][v] = 2.0 * (g + k) * ginv;    /* g2 */
    b->cf[2][v] = g * ginv;                /* g3 */
    b->cf[3][v] = 2.0 * ginv;              /* g4 */
    b->cf[4][v] = k;
}

/* maxiBiquad::set, src/maximilian.h:1375-1479. abs() there resolves to the double overload. */
static void biquad_set(const bank_t* b, int v) {
    const double sr = (double)(size_t)b->chain.sample_rate;
    const double cutoff = b->p[MXO_P_CUTOFF][v], Q = b->p[MXO_P_RESONANCE][v], peakGain = b->p[MXO_P_GAIN][v];
    const double SQRT2 = sqrt(2.0);                      /* src/maximilian.h:1484 */
    double norm = 0, a0 = 0, a1 = 0, a2 = 0, b1 = 0, b2 = 0;
    const double Vg = pow(10.0, fabs(peakGain) / 20.0);
    const double K = tan(MAXI_PI * cutoff / sr);
    switch (b->chain.biquad_type) {
        case 0: /* LOWPASS :1381-1388 */
            norm = 1.0 / (1.0 + K / Q + K * K);
            a0 = K * K * norm; a1 = 2.0 * a0; a2 = a0;
            b1 = 2.0 * (K * K - 1.0) * norm; b2 = (1.0 - K / Q + K * K) * norm; break;
        case 1: /* HIGHPASS :1390-1397 */
            norm = 1. / (1. + K / Q + K * K);
            a0 = 1 * norm; a1 = -2 * a0; a2 = a0;
            b1 = 2 * (K * K - 1) * norm; b2 = (1 - K / Q + K * K) * norm; break;
        case 2: /* BANDPASS :1399-1406 */
            norm = 1. / (1. + K / Q + K * K);
            a0 = K / Q * norm; a1 = 0.; a2 = -a0;
            b1 = 2. * (K * K - 1.) * norm; b2 = (1. - K / Q + K * K) * norm; break;
        case 3: /* NOTCH :1408-1415 */
            norm = 1. / (1. + K / Q + K * K);
            a0 = (1. + K * K) * norm; a1 = 2. * (K * K - 1.) * norm; a2 = a0;
            b1 = a1; b2 = (1. - K / Q + K * K) * norm; break;
        case 4: /* PEAK :1417-1436 */
            if (peakGain >= 0.0) {
                norm = 1. / (1. + 1. / Q * K + K * K);
                a0 = (1. + Vg / Q * K + K * K) * norm; a1 = 2. * (K * K - 1.) * norm;
                a2 = (1. - Vg / Q * K + K * K) * norm; b1 = a1; b2 = (1. - 1. / Q * K + K * K) * norm;
            } else {
                norm = 1. / (1. + Vg / Q * K + K * K);
                a0 = (1. + 1 / Q * K + K * K) * norm; a1 = 2. * (K * K - 1) * norm;
                a2 = (1. - 1. / Q * K + K * K) * norm; b1 = a1; b2 = (1. - Vg / Q * K + K * K) * norm;
            }
            break;
        case 5: /* LOWSHELF :1437-1456 */
            if (peakGain >= 0.) {
                norm = 1. / (1. + SQRT2 * K + K * K);
                a0 = (1. + sqrt(2. * Vg) * K + Vg * K * K) * norm; a1 = 2. * (Vg * K * K - 1.) * norm;
                a2 = (1. - sqrt(2. * Vg) * K + Vg * K * K) * norm;
                b1 = 2. * (K * K - 1.) * norm; b2 = (1. - SQRT2 * K + K * K) * norm;
            } else {
                norm = 1. / (1. + sqrt(2. * Vg) * K + Vg * K * K);
                a0 = (1. + SQRT2 * K + K * K) * norm; a1 = 2. * (K * K - 1.) * norm;
                a2 = (1. - SQRT2 * K + K * K) * norm;
                b1 = 2. * (Vg * K * K - 1.) * norm; b2 = (1. - sqrt(2. * Vg) * K + Vg * K * K) * norm;
            }
            break;
        case 6: /* HIGHSHELF :1457-1476 */
            if (peakGain >= 0.) {
                norm = 1. / (1. + SQRT2 * K + K * K);
                a0 = (Vg + sqrt(2. * Vg) * K + K * K) * norm; a1 = 2. * (K * K - Vg) * norm;
                a2 = (Vg - sqrt(2. * Vg) * K + K * K) * norm;
                b1 = 2. * (K * K - 1) * norm; b2 = (1. - SQRT2 * K + K * K) * norm;
            } else {
                norm = 1. / (Vg + sqrt(2. * Vg) * K + K * K);
                a0 = (1. + SQRT2 * K + K * K) * norm; a1 = 2. * (K * K - 1.) * norm;
                a2 = (1. - SQRT2 * K + K * K) * norm;
                b1 = 2. * (K * K - Vg) * norm; b2 = (Vg - sqrt(2. * Vg) * K + K * K) * norm;
            }
            break;
        default: break;
    }
    b->cf[0][v] = a0; b->cf[1][v] = a1; b->cf[2][v] = a2; b->cf[3][v] = b1; b->cf[4][v] = b2;
}

void* mxo_bank_create(const mxo_chain* chain, int32_t voices) {
    if (!chain || voices <= 0) return NULL;
    bank_t* b = (bank_t*)calloc(1, sizeof(bank_t));
    if (!b) return NULL;
    const size_t V = (size_t)voices;
    b->chain = *chain;
    b->V = voices;
    for (int i = 0; i < MXO_P_COUNT; ++i) b->p[i] = dalloc(V, 0.0);
    for (size_t v = 0; v < V; ++v) {
        b->p[MXO_P_DUTY][v] = 0.5; b->p[MXO_P_DELAY_SIZE][v] = 1.0; b->p[MXO_P_PAN][v] = 0.5; b->p[MXO_P_PHASOR_END][v] = 1.0;
        b->p[MXO_P_ENV_HOLDTIME][v] = 1.0;          /* src/maximilian.h:913 */
        b->p[MXO_P_CUTOFF][v] = 1000.0; b->p[MXO_P_RESONANCE][v] = 1.0;   /* maxiSVF ctor, src/maximilian.h:1284 */
    }
    b->osc_out = dalloc(V, 0.0);
    b->f0 = dalloc(V, 0.0); b->f1 = dalloc(V, 0.0); b->f2 = dalloc(V, 0.0);
    for (int i = 0; i < 5; ++i) b->cf[i] = dalloc(V, 0.0);   /* maxiBiquad coefficients default to 0, src/maximilian.h:1482 */
    b->env_amp = dalloc(V, 0.0); b->env_output = dalloc(V, 0.0);
    b->env_holdcount = (int64_t*)calloc(V, sizeof(int64_t));
    b->env_flags = (int32_t*)calloc(V, sizeof(int32_t));
    b->dl_phase = (int32_t*)calloc(V, sizeof(int32_t));
    if (chain->filt_kind == MXO_FILT_SVF) for (int v = 0; v < voices; ++v) svf_set_params(b, v);
    if (chain->delay_on) {
        if (chain->delay_capacity <= 0) { free(b); return NULL; }
        b->ring = (double*)calloc(V * (size_t)chain->delay_capacity, sizeof(double));  /* ctor memset, src/maximilian.cpp:415-417 */
        if (!b->ring) { free(b); return NULL; }
    }
    return b;
}

void mxo_bank_destroy(void* h) {
    bank_t* b = (bank_t*)h;
    if (!b) return;
    for (int i = 0; i < 16; ++i) free(b->p[i]);
    free(b->osc_out); free(b->f0); free(b->f1); free(b->f2);
    for (int i = 0; i < 5; ++i) free(b->cf[i]);
    free(b->env_amp); free(b->env_output); free(b->env_holdcount); free(b->env_flags);
    free(b->dl_phase); free(b->ring); free(b);
}

int32_t mxo_bank_set(void* h, int32_t id, const double* x) {
    bank_t* b = (bank_t*)h;
    if (!b || !x || id < 0 || id >= MXO_P_COUNT) return -1;
    memcpy(b->p[id], x, sizeof(double) * (size_t)b->V);
    if (id == MXO_P_CUTOFF || id == MXO_P_RESONANCE || id == MXO_P_GAIN) {
        if (b->chain.filt_kind == MXO_FILT_SVF) for (int v = 0; v < b->V; ++v) svf_set_params(b, v);
        if (b->chain.filt_kind == MXO_FILT_BIQUAD) for (int v = 0; v < b->V; ++v) biquad_set(b, v);
    }
    return 0;
}

int32_t mxo_bank_get(void* h, int32_t id, double* x) {
    bank_t* b = (bank_t*)h;
    if (!b || !x) return -1;
    for (int v = 0; v < b->V; ++v) {
        switch (id) {
            case MXO_S_FILT_0: x[v] = b->f0[v]; break;
            case MXO_S_FILT_1: x[v] = b->f1[v]; break;
            case MXO_S_FILT_2: x[v] = b->chain.filt_kind == MXO_FILT_SVF ? b->f2[v] : 0.0; break;
            case MXO_S_ENV_AMPLITUDE: x[v] = b->env_amp[v]; break;
            case MXO_S_ENV_OUTPUT: x[v] = b->env_output[v]; break;
            case MXO_S_ENV_HOLDCOUNT: x[v] = (double)b->env_holdcount[v]; break;
            case MXO_S_ENV_FLAGS: x[v] = (double)b->env_flags[v]; break;
            case MXO_S_DELAY_PHASE: x[v] = (double)b->dl_phase[v]; break;
            case MXO_S_OSC_OUTPUT: x[v] = b->osc_out[v]; break;
            default: if (id >= 0 && id < MXO_P_COUNT) x[v] = b->p[id][v]; else return -1;
        }
    }
    return 0;
}

int32_t mxo_bank_get_ring(void* h, int32_t v, double* dst, int32_t n) {
    bank_t* b = (bank_t*)h;
    if (!b || !b->ring || v < 0 || v >= b->V || n < 0 || n > b->chain.delay_capacity) return -1;
    memcpy(dst, b->ring + (size_t)v * (size_t)b->chain.delay_capacity, sizeof(double) * (size_t)n);
    return 0;
}

/* maxiOsc::*, src/maximilian.cpp:228-235 (sinewave), 276-283 (coswave), 285-291 (phasor),
 * 293-300 (square), 302-311 (pulse), 312-319 (impulse), 321-330 (phasorBetween), 333-340 (saw), 362-373 (triangle).
 * The increment is 1./(sampleRate/frequency) with sampleRate a size_t: two divides, kept. */
static inline double osc_tick(int kind, double* phase_p, double* output_p, double frequency, double duty, double sr,
                              double startphase, double endphase) {
    double phase = *phase_p, output = *output_p;
    switch (kind) {
        case MXO_OSC_SINEWAVE:
            output = sin(phase * (MAXI_TWOPI));
            if (phase >= 1.0) phase -= 1.0;
            phase += (1. / (sr / (frequency)));
            break;
        case MXO_OSC_COSWAVE:
            output = cos(phase * (MAXI_TWOPI));
            if (phase >= 1.0) phase -= 1.0;
            phase += (1. / (sr / (frequency)));
            break;
        case MXO_OSC_PHASOR:
            output = phase;
            if (phase >= 1.0) phase -= 1.0;
            phase += (1. / (sr / (frequency)));
            break;
        case MXO_OSC_SAW:
            output = phase;
            if (phase >= 1.0) phase -= 2.0;
            phase += (1. / (sr / (frequency))) * 2.0;
            break;
        case MXO_OSC_SQUARE:
            if (phase < 0.5) output = -1;
            if (phase > 0.5) output = 1;
            if (phase >= 1.0) phase -= 1.0;
            phase += (1. / (sr / (frequency)));
            break;
        case MXO_OSC_PULSE:
            if (duty < 0.) duty = 0;
            if (duty > 1.) duty = 1;
            if (phase >= 1.0) phase -= 1.0;
            phase += (1. / (sr / (frequency)));
            if (phase < duty) output = -1.;
            if (phase > duty) output = 1.;
            break;
        case MXO_OSC_IMPULSE: {
            if (phase >= 1.0) phase -= 1.0;
            double phaseInc = (1. / (sr / (frequency)));
            double o = phase < phaseInc ? 1.0 : 0.0;     /* a local in the reference: the member is untouched */
            phase += phaseInc;
            *phase_p = phase;
            return o;
        }
        case MXO_OSC_TRIANGLE:
            if (phase >= 1.0) phase -= 1.0;
            phase += (1. / (sr / (frequency)));
            if (phase <= 0.5) output = (phase - 0.25) * 4;
            else output = ((1.0 - phase) - 0.25) * 4;
            break;
        case MXO_OSC_PHASORBETWEEN:
            output = phase;
            if (phase < startphase) {
                phase = startphase;
            }
            if (phase >= endphase) phase = startphase;
            phase += ((endphase - startphase) / (sr / (frequency)));
            break;
        default: break;
    }
    *phase_p = phase; *output_p = output;
    return output;
}

/* maxiEnv::adsr(double input, int trigger), src/maximilian.cpp:1415-1466 */
static inline double env_adsr(bank_t* b, int v, double input, int trigger) {
    int fl = b->env_flags[v];
    int attackphase = fl & 1, decayphase = (fl >> 1) & 1, sustainphase = (fl >> 2) & 1,
        holdphase = (fl >> 3) & 1, releasephase = (fl >> 4) & 1;
    double amplitude = b->env_amp[v], output = b->env_output[v];
    int64_t holdcount = b->env_holdcount[v];
    const double attack = b->p[MXO_P_ENV_ATTACK][v], decay = b->p[MXO_P_ENV_DECAY][v],
                 sustain = b->p[MXO_P_ENV_SUSTAIN][v], release = b->p[MXO_P_ENV_RELEASE][v];
    const int64_t holdtime = (int64_t)b->p[MXO_P_ENV_HOLDTIME][v];

    if (trigger == 1 && attackphase != 1 && holdphase != 1 && decayphase != 1) {
        holdcount = 0; decayphase = 0; sustainphase = 0; releasephase = 0; attackphase = 1;
    }
    if (attackphase == 1) {
        releasephase = 0;
        amplitude += (1 * attack);
        output = input * amplitude;
        if (amplitude >= 1) { amplitude = 1; attackphase = 0; decayphase = 1; }
    }
    if (decayphase == 1) {
        output = input * (amplitude *= decay);
        if (amplitude <= sustain) { decayphase = 0; holdphase = 1; }
    }
    if (holdcount < holdtime && holdphase == 1) { output = input * amplitude; holdcount++; }
    if (holdcount >= holdtime && trigger == 1) { output = input * amplitude; }
    if (holdcount >= holdtime && trigger != 1) { holdphase = 0; releasephase = 1; }
    if (releasephase == 1 && amplitude > 0.) { output = input * (amplitude *= release); }

    b->env_flags[v] = attackphase | decayphase << 1 | sustainphase << 2 | holdphase << 3 | releasephase << 4;
    b->env_amp[v] = amplitude; b->env_output[v] = output; b->env_holdcount[v] = holdcount;
    return output;
}

/* maxiEnv::ar(input, attack, release, holdtime, trigger), src/maximilian.cpp:1319-1358 (the arguments come from the
 * per-voice attack / release / holdtime arrays) */
static inline double env_ar(bank_t* b, int v, double input, int trigger) {
    int fl = b->env_flags[v];
    int attackphase = fl & 1, decayphase = (fl >> 1) & 1, sustainphase = (fl >> 2) & 1,
        holdphase = (fl >> 3) & 1, releasephase = (fl >> 4) & 1;
    double amplitude = b->env_amp[v], output = b->env_output[v];
    int64_t holdcount = b->env_holdcount[v];
    const double attack = b->p[MXO_P_ENV_ATTACK][v], release = b->p[MXO_P_ENV_RELEASE][v];
    const int64_t holdtime = (int64_t)b->p[MXO_P_ENV_HOLDTIME][v];

    if (trigger == 1 && attackphase != 1 && holdphase != 1) { holdcount = 0; releasephase = 0; attackphase = 1; }
    if (attackphase == 1) { amplitude += (1 * attack); output = input * amplitude; }
    if (amplitude >= 1) { amplitude = 1; attackphase = 0; holdphase = 1; }
    if (holdcount < holdtime && holdphase == 1) { output = input; holdcount++; }
    if (holdcount == holdtime && trigger == 1) { output = input; }
    if (holdcount == holdtime && trigger != 1) { holdphase = 0; releasephase = 1; }
    if (releasephase == 1 && amplitude > 0.) { output = input * (amplitude *= release); }

    b->env_flags[v] = attackphase | decayphase << 1 | sustainphase << 2 | holdphase << 3 | releasephase << 4;
    b->env_amp[v] = amplitude; b->env_output[v] = output; b->env_holdcount[v] = holdcount;
    return output;
}

int32_t mxo_bank_process(void* h, int32_t nframes, const int32_t* trig_on, const int32_t* trig_off,
                         double* out, double* mix, int32_t first, int32_t count) {
    return mxo_bank_process_fm(h, nframes, NULL, trig_on, trig_off, out, mix, first, count);
}

int32_t mxo_bank_process_fm(void* h, int32_t nframes, const double* freq_tv, const int32_t* trig_on, const int32_t* trig_off,
                            double* out, double* mix, int32_t first, int32_t count) {
    return mxo_bank_process_mod(h, nframes, freq_tv, NULL, NULL, trig_on, trig_off, out, mix, first, count);
}

int32_t mxo_bank_process_mod(void* h, int32_t nframes, const double* freq_tv, const double* cutoff_tv, const double* delay_size_tv,
                             const int32_t* trig_on, const int32_t* trig_off, double* out, double* mix, int32_t first, int32_t count) {
    return mxo_bank_process_mod2(h, nframes, freq_tv, cutoff_tv, delay_size_tv, NULL, trig_on, trig_off, out, mix, first, count);
}

/* ... and with the envelope's trigger given for every sample: trig_tv[t][v] bytes, maxiEnv::trigger as the patch sets it before each
 * call (src/maximilian.h:913; cpp/commandline/maximilian_examples/10.Filters/main.cpp:27-36) */
int32_t mxo_bank_process_mod2(void* h, int32_t nframes, const double* freq_tv, const double* cutoff_tv, const double* delay_size_tv,
                              const uint8_t* trig_tv, const int32_t* trig_on, const int32_t* trig_off, double* out, double* mix, int32_t first, int32_t count) {
    bank_t* b = (bank_t*)h;
    if (!b || nframes < 0 || first < 0 || count < 0 || first + count > b->V) return -1;
    const mxo_chain* c = &b->chain;
    const int V = b->V;
    const double sr = (double)(size_t)c->sample_rate;     /* maxiSettings::sampleRate is a size_t, src/maximilian.h:124 */
    if (cutoff_tv && c->filt_kind == MXO_FILT_BIQUAD) return -3;
    if (delay_size_tv && !c->delay_on) return -3;
    for (int t = 0; t < nframes; ++t) {
        double m0 = 0.0, m1 = 0.0;
        for (int v = first; v < first + count; ++v) {
            /* the reference takes the frequency by argument on every call: a patch may pass a new one each sample
             * (FM: maximilian_examples/5.FM1/main.cpp:29) */
            const double fq = freq_tv ? freq_tv[(size_t)t * (size_t)V + (size_t)v] : b->p[MXO_P_FREQ][v];
            double x = osc_tick(c->osc_kind, &b->p[MXO_P_PHASE][v], &b->osc_out[v], fq, b->p[MXO_P_DUTY][v], sr,
                                b->p[MXO_P_PHASOR_START][v], b->p[MXO_P_PHASOR_END][v]);
            if (c->env_kind == MXO_ENV_ADSR) {
                int trig = trig_tv ? (int)trig_tv[(size_t)t * (size_t)V + (size_t)v] : (trig_on && trig_off && t >= trig_on[v] && t < trig_off[v]) ? 1 : 0;
                x = env_adsr(b, v, x, trig);
            } else if (c->env_kind == MXO_ENV_AR) {
                int trig = trig_tv ? (int)trig_tv[(size_t)t * (size_t)V + (size_t)v] : (trig_on && trig_off && t >= trig_on[v] && t < trig_off[v]) ? 1 : 0;
                x = env_ar(b, v, x, trig);
            }
            switch (c->filt_kind) {
                case MXO_FILT_LORES:
                case MXO_FILT_HIRES: {
                    /* maxiFilter::lores / hires, src/maximilian.cpp:455-468 / 471-484 */
                    double input = x, resonance = b->p[MXO_P_RESONANCE][v];
                    double cutoff = cutoff_tv ? cutoff_tv[(size_t)t * (size_t)V + (size_t)v] : b->p[MXO_P_CUTOFF][v];
                    double fx = b->f0[v], fy = b->f1[v];
                    if (cutoff < 10) cutoff = 10;
                    if (cutoff > sr) cutoff = sr;
                    if (resonance < 1.) resonance = 1.;
                    double z = cos(MAXI_TWOPI * cutoff / sr);
                    double cc = 2 - 2 * z;
                    double r = (sqrt(2.0) * sqrt(-pow((z - 1.0), 3.0)) + resonance * (z - 1)) / (resonance * (z - 1));
                    fx = fx + (input - fy) * cc;
                    fy = fy + fx;
                    fx = fx * r;
                    b->f0[v] = fx; b->f1[v] = fy;
                    x = (c->filt_kind == MXO_FILT_LORES) ? fy : input - fy;
                    break;
                }
                case MXO_FILT_SVF: {
                    /* maxiSVF::play, src/maximilian.h:1305-1319 */
                    double g1 = b->cf[0][v], g2 = b->cf[1][v], g3 = b->cf[2][v], g4 = b->cf[3][v], k = b->cf[4][v];
                    if (cutoff_tv) {
                        /* maxiSVF::setCutoff -> setParams(cutoff, res), src/maximilian.h:1287-1290,1322-1334, called by
                         * the patch before play(); the object's own members keep MXO_P_CUTOFF for the calls after this one */
                        const double freq = cutoff_tv[(size_t)t * (size_t)V + (size_t)v], res = b->p[MXO_P_RESONANCE][v];
                        const double g = tan(MAXI_PI * freq / sr);
                        const double damping = res == 0 ? 0 : 1.0 / res;
                        const double ginv = g / (1.0 + g * (g + damping));
                        k = damping;
                        g1 = ginv; g2 = 2.0 * (g + k) * ginv; g3 = g * ginv; g4 = 2.0 * ginv;
                    }
                    double w = x, v0z = b->f0[v], v1 = b->f1[v], v2 = b->f2[v];
                    double low, band, high, notch;
                    double v1z = v1;
                    double v2z = v2;
                    double v3 = w + v0z - 2.0 * v2z;
                    v1 += g1 * v3 - g2 * v1z;
                    v2 += g3 * v3 + g4 * v1z;
                    v0z = w;
                    low = v2;
                    band = v1;
                    high = w - k * v1 - v2;
                    notch = w - k * v1;
                    b->f0[v] = v0z; b->f1[v] = v1; b->f2[v] = v2;
                    x = (low * c->svf_mix[0]) + (band * c->svf_mix[1]) + (high * c->svf_mix[2]) + (notch * c->svf_mix[3]);
                    break;
                }
                case MXO_FILT_BIQUAD: {
                    /* maxiBiquad::play, src/maximilian.h:1360-1367 */
                    const double a0 = b->cf[0][v], a1 = b->cf[1][v], a2 = b->cf[2][v], b1 = b->cf[3][v], b2 = b->cf[4][v];
                    double v1 = b->f0[v], v2 = b->f1[v];
                    double v0 = x - (b1 * v1) - (b2 * v2);
                    double y = (a0 * v0) + (a1 * v1) + (a2 * v2);
                    b->f1[v] = v1; b->f0[v] = v0;
                    x = y;
                    break;
                }
                default: break;
            }
            if (c->delay_on) {
                /* maxiDelayline::dl, src/maximilian.cpp:420-429 */
                /* `size` is an int argument of every call: a flanger passes a new one each sample (double -> int conversion) */
                const int size = delay_size_tv ? (int)delay_size_tv[(size_t)t * (size_t)V + (size_t)v] : (int)b->p[MXO_P_DELAY_SIZE][v];
                const double feedback = b->p[MXO_P_DELAY_FEEDBACK][v];
                double* memory = b->ring + (size_t)v * (size_t)c->delay_capacity;
                int phase = b->dl_phase[v];
                if (phase >= size) phase = 0;
                if (phase < 0 || phase >= c->delay_capacity) return -4;   /* the reference would index out of its 705600 slots */
                double output;
                if (c->delay_on == 2) {
                    /* maxiDelayline::dlFromPosition, src/maximilian.cpp:431-439; chandiv (src/maximilian.cpp:53) is the float 1 */
                    int position = (int)b->p[MXO_P_DELAY_POSITION][v];
                    if (position >= size) position = 0;
                    if (position < 0 || position >= c->delay_capacity) return -4;
                    output = memory[position];
                    memory[phase] = (memory[phase] * feedback) + (x * feedback) * 1.0f;
                } else {
                    output = memory[phase];
                    memory[phase] = (memory[phase] * feedback) + (x * feedback) * 0.5;
                }
                phase += 1;
                b->dl_phase[v] = phase;
                x = output;
            }
            if (out) out[(size_t)t * (size_t)V + (size_t)v] = x;
            if (mix) {
                /* maxiMix::stereo, src/maximilian.cpp:503-509 */
                double px = b->p[MXO_P_PAN][v];
                if (px > 1) px = 1;
                if (px < 0) px = 0;
                m0 += x * sqrt(1.0 - px);
                m1 += x * sqrt(px);
            }
        }
        if (mix) { mix[2 * t] = m0; mix[2 * t + 1] = m1; }
    }
    return 0;
}

/* maxiEnv::setAttack / setAttackMS / setDecay (= setRelease), src/maximilian.cpp:1469-1486 */
double mxo_env_attack_coeff(double attackMS, int32_t sr) { return 1 - pow(0.01, 1.0 / (attackMS * (double)(size_t)sr * 0.001)); }
double mxo_env_attack_ms_coeff(double attackMS, int32_t sr) { return 1.0 / (attackMS / 1000.0 * (double)(size_t)sr); }
double mxo_env_decay_coeff(double ms, int32_t sr) { return pow(0.01, 1.0 / (ms * (double)(size_t)sr * 0.001)); }

/* ================================================================= patches
 * A patch is a per-voice signal graph: the body of a reference play() as a list of stages over 16 registers
 * (oracle_api.h). Every stage body below restates one reference method; state lives in st[] slots per (stage, voice). */

static double g_sine[514], g_transition[1001], g_sine_before = 0.0;
static int g_tables_set = 0;

/* sineBuffer / transition (src/maximilian.cpp:63, 67-200) are data of the reference: they are handed in at run time
 * (from the compiled reference, or from tests/golden/tables.npz), never copied into this file. sine_before: the double
 * sinebuf4 reads at sineBuffer[-1] on its wrap sample (an out-of-bounds read in the reference). */
int32_t mxo_set_tables(const double* sine514, const double* transition1001, double sine_before) {
    if (!sine514 || !transition1001) return -1;
    memcpy(g_sine, sine514, sizeof(g_sine)); memcpy(g_transition, transition1001, sizeof(g_transition));
    g_sine_before = sine_before; g_tables_set = 1;
    return 0;
}
int32_t mxo_get_tables(double* sine514, double* transition1001, double* sine_before) {
    if (!g_tables_set) return -1;
    memcpy(sine514, g_sine, sizeof(g_sine)); memcpy(transition1001, g_transition, sizeof(g_transition));
    *sine_before = g_sine_before;
    return 0;
}

typedef struct { double startlevel, endlevel, currentlevel, gradient, curve; size_t length, counter; int hold; } eg_stage_t;
typedef struct { eg_stage_t seg[MXO_MAX_EG_SEGMENTS]; int n, loop, retrigger; } eg_shape_t;    /* one maxiEnvGen after setup() */

typedef struct {
    mxo_patch_desc d;
    mxo_stage* stages;
    double* consts;
    int* sbase; int* ringof;
    int n_state, n_rings;
    double* params;   /* [n_params][V] */
    double* state;    /* [n_state][V] */
    double* rings;    /* [n_rings][V][taps] */
    double reg[16];
    eg_shape_t eg[MXO_MAX_EG_SHAPES];
} patch_t;

static int p_state_slots(const mxo_stage* g) {
    switch (g->op) {
        case MXO_OP_OSC: return 2;
        case MXO_OP_ENV_ADSR: case MXO_OP_ENV_AR: return 4;
        case MXO_OP_ENVGEN: return 12;
        case MXO_OP_FILTER: return 2;
        case MXO_OP_SVF: return 3;
        case MXO_OP_BIQUAD: return 2;
        case MXO_OP_DCBLOCK: return 2;
        case MXO_OP_DELAY: return 1;
        case MXO_OP_FLANGER: return 3;
        case MXO_OP_CHORUS: return 4;
        default: return 0;
    }
}
static int p_stage_rings(const mxo_stage* g) { return g->op == MXO_OP_CHORUS ? 2 : (g->op == MXO_OP_DELAY || g->op == MXO_OP_FLANGER) ? 1 : 0; }

/* maxiOsc::noise, src/maximilian.cpp:214-220, on libc rand() */
void mxo_srand(uint32_t seed) { srand(seed); }
void mxo_noise_fill(uint32_t seed, int64_t n, double* out) {
    srand(seed);
    for (int64_t i = 0; i < n; ++i) { float r = rand() / (float)RAND_MAX; out[i] = r * 2 - 1; }
}

void* mxo_patch_create(const mxo_patch_desc* d) {
    if (!d || d->voices <= 0 || d->n_stages <= 0 || d->n_stages > 64 || !d->stages || !mxo_patch_shapes_ok(d)) return NULL;
    patch_t* p = (patch_t*)calloc(1, sizeof(patch_t));
    p->d = *d;
    p->d.shapes = NULL;                                    /* copied into p->eg below */
    p->stages = (mxo_stage*)malloc(sizeof(mxo_stage) * (size_t)d->n_stages);
    memcpy(p->stages, d->stages, sizeof(mxo_stage) * (size_t)d->n_stages);
    p->consts = (double*)calloc(64, sizeof(double));
    if (d->n_consts) memcpy(p->consts, d->consts, sizeof(double) * (size_t)d->n_consts);
    p->sbase = (int*)calloc((size_t)d->n_stages, sizeof(int)); p->ringof = (int*)calloc((size_t)d->n_stages, sizeof(int));
    for (int i = 0; i < d->n_stages; ++i) {
        p->sbase[i] = p->n_state; p->n_state += p_state_slots(&p->stages[i]);
        const int nr = p_stage_rings(&p->stages[i]);
        p->ringof[i] = nr ? p->n_rings : -1;
        p->n_rings += nr;
    }
    const size_t V = (size_t)d->voices;
    p->params = (double*)calloc((size_t)(d->n_params ? d->n_params : 1) * V, sizeof(double));
    p->state = (double*)calloc((size_t)(p->n_state ? p->n_state : 1) * V, sizeof(double));
    if (p->n_rings) p->rings = (double*)calloc((size_t)p->n_rings * V * (size_t)d->delay_taps, sizeof(double));
    /* maxiTrigger: previousValue = 1, firstTrigger = 1 (src/maximilian.h:583-584) */
    for (int i = 0; i < d->n_stages; ++i)
        if (p->stages[i].op == MXO_OP_ENVGEN)
            for (int k = 6; k < 12; ++k) for (size_t v = 0; v < V; ++v) p->state[(size_t)(p->sbase[i] + k) * V + v] = 1.0;
    /* maxiEnvGen::setup / setupSegmentTime, src/maximilian.h:2371-2402, 2524-2538, once per shape: each is its own object */
    for (int k = 0; k < d->n_shapes; ++k) {
        const mxo_envgen_shape* sh = &d->shapes[k];
        eg_shape_t* e = &p->eg[k];
        e->n = sh->stages; e->loop = sh->loop; e->retrigger = sh->retrigger;
        double accumulatedTime = 0;
        const double sr = (double)(size_t)d->sample_rate;
        for (int i = 0; i < sh->stages; ++i) {
            eg_stage_t* s = &e->seg[i];
            s->startlevel = sh->levels[i]; s->endlevel = sh->levels[i + 1];
            const double stageTime = sh->times[i];
            if (stageTime == MXO_ENVGEN_HOLD) { s->length = 0; s->hold = 1; s->gradient = 0; }
            else {
                double len = ((stageTime / 1000.0) * sr) + accumulatedTime;
                s->length = (size_t)floor(len);
                accumulatedTime = len - s->length;
                s->gradient = 1.0 / s->length;
                s->hold = 0;
            }
            s->curve = sh->curves[i]; s->counter = 0; s->currentlevel = 0;
        }
    }
    return p;
}

void mxo_patch_destroy(void* h) {
    patch_t* p = (patch_t*)h; if (!p) return;
    free(p->stages); free(p->consts); free(p->sbase); free(p->ringof); free(p->params); free(p->state); free(p->rings); free(p);
}

int32_t mxo_patch_set_param(void* h, int32_t j, const double* x) {
    patch_t* p = (patch_t*)h; if (!p || !x || j < 0 || j >= p->d.n_params) return -1;
    memcpy(p->params + (size_t)j * (size_t)p->d.voices, x, sizeof(double) * (size_t)p->d.voices);
    return 0;
}
int32_t mxo_patch_set_state(void* h, int32_t stage, int32_t slot, const double* x) {
    patch_t* p = (patch_t*)h; if (!p || !x || stage < 0 || stage >= p->d.n_stages || slot < 0 || slot >= p_state_slots(&p->stages[stage])) return -1;
    memcpy(p->state + (size_t)(p->sbase[stage] + slot) * (size_t)p->d.voices, x, sizeof(double) * (size_t)p->d.voices);
    return 0;
}
int32_t mxo_patch_get_state(void* h, int32_t stage, int32_t slot, double* x) {
    patch_t* p = (patch_t*)h; if (!p || !x || stage < 0 || stage >= p->d.n_stages || slot < 0 || slot >= p_state_slots(&p->stages[stage])) return -1;
    memcpy(x, p->state + (size_t)(p->sbase[stage] + slot) * (size_t)p->d.voices, sizeof(double) * (size_t)p->d.voices);
    return 0;
}
int32_t mxo_patch_get_ring(void* h, int32_t stage, int32_t v, double* dst, int32_t n) {
    patch_t* p = (patch_t*)h;
    if (!p || !dst || stage < 0 || stage >= p->d.n_stages || p->ringof[stage] < 0 || v < 0 || v >= p->d.voices || n < 0) return -1;
    const int taps = p->d.delay_taps, nr = p_stage_rings(&p->stages[stage]);
    if (n > taps * nr) return -1;
    for (int k = 0; k < nr && k * taps < n; ++k) {          /* a chorus stage's two lines back to back */
        const int m = n - k * taps < taps ? n - k * taps : taps;
        memcpy(dst + (size_t)k * taps, p->rings + ((size_t)(p->ringof[stage] + k) * (size_t)p->d.voices + (size_t)v) * (size_t)taps, sizeof(double) * (size_t)m);
    }
    return 0;
}

/* maxiOsc::sinebuf4 / sinebuf / sawn, src/maximilian.cpp:237-274, 342-359 */
static double p_osc_table(int kind, double* phase_p, double* output_p, double frequency, double sr) {
    double phase = *phase_p, output;
    if (kind == MXO_OSC_SINEBUF4) {
        double remainder, a, b, c, d, a1, a2, a3;
        phase += 512. / (sr / (frequency));
        if (phase >= 511) phase -= 512;
        remainder = phase - floor(phase);
        if (phase == 0) {
            a = g_sine[(long)512]; b = g_sine[(long)phase]; c = g_sine[(long)phase + 1]; d = g_sine[(long)phase + 2];
        } else {
            a = ((long)phase - 1 < 0) ? g_sine_before : g_sine[(long)phase - 1];
            b = g_sine[(long)phase]; c = g_sine[(long)phase + 1]; d = g_sine[(long)phase + 2];
        }
        a1 = 0.5f * (c - a);
        a2 = a - 2.5 * b + 2.f * c - 0.5f * d;
        a3 = 0.5f * (d - a) + 1.5f * (b - c);
        output = (double)(((a3 * remainder + a2) * remainder + a1) * remainder + b);
    } else if (kind == MXO_OSC_SINEBUF) {
        double remainder;
        phase += 512. / (sr / (frequency * 1.0f));          /* chandiv == 1, src/maximilian.cpp:53 */
        if (phase >= 511) phase -= 512;
        remainder = phase - floor(phase);
        output = (double)((1 - remainder) * g_sine[1 + (long)phase] + remainder * g_sine[2 + (long)phase]);
    } else {
        if (phase >= 0.5) phase -= 1.0;
        phase += (1. / (sr / (frequency)));
        double temp = (8820.22 / frequency) * phase;
        if (temp < -0.5) temp = -0.5;
        if (temp > 0.5) temp = 0.5;
        temp *= 1000.0f;
        temp += 500.0f;
        double remainder = temp - floor(temp);
        /* transition[1 + (long)temp] is one past the table when temp == 1000; remainder is 0 there */
        double t1 = (1 + (long)temp <= 1000) ? g_transition[1 + (long)temp] : 0.0;
        output = (double)((1.0f - remainder) * g_transition[(long)temp] + remainder * t1) - phase;
    }
    *phase_p = phase; *output_p = output;
    return output;
}

/* maxiEnv::adsr(input, attack, decay, sustain, release, holdtime, trigger), src/maximilian.cpp:1362-1413 (the same
 * state machine as the member-parameter overload :1415-1466); st = amplitude, output, holdcount, flags */
static double p_env_adsr(double* st, size_t V, double input, int trigger, double attack, double decay, double sustain, double release, long holdtime) {
    double amplitude = st[0], output = st[V];
    long holdcount = (long)st[2 * V];
    int fl = (int)st[3 * V];
    int attackphase = fl & 1, decayphase = (fl >> 1) & 1, sustainphase = (fl >> 2) & 1, holdphase = (fl >> 3) & 1, releasephase = (fl >> 4) & 1;
    if (trigger == 1 && attackphase != 1 && holdphase != 1 && decayphase != 1) {
        holdcount = 0; decayphase = 0; sustainphase = 0; releasephase = 0; attackphase = 1;
    }
    if (attackphase == 1) {
        releasephase = 0;
        amplitude += (1 * attack);
        output = input * amplitude;
        if (amplitude >= 1) { amplitude = 1; attackphase = 0; decayphase = 1; }
    }
    if (decayphase == 1) {
        output = input * (amplitude *= decay);
        if (amplitude <= sustain) { decayphase = 0; holdphase = 1; }
    }
    if (holdcount < holdtime && holdphase == 1) { output = input * amplitude; holdcount++; }
    if (holdcount >= holdtime && trigger == 1) { output = input * amplitude; }
    if (holdcount >= holdtime && trigger != 1) { holdphase = 0; releasephase = 1; }
    if (releasephase == 1 && amplitude > 0.) { output = input * (amplitude *= release); }
    st[0] = amplitude; st[V] = output; st[2 * V] = (double)holdcount;
    st[3 * V] = (double)(attackphase | decayphase << 1 | sustainphase << 2 | holdphase << 3 | releasephase << 4);
    return output;
}

/* maxiEnv::ar, src/maximilian.cpp:1319-1358 */
static double p_env_ar(double* st, size_t V, double input, int trigger, double attack, double release, long holdtime) {
    double amplitude = st[0], output = st[V];
    long holdcount = (long)st[2 * V];
    int fl = (int)st[3 * V];
    int attackphase = fl & 1, decayphase = (fl >> 1) & 1, sustainphase = (fl >> 2) & 1, holdphase = (fl >> 3) & 1, releasephase = (fl >> 4) & 1;
    if (trigger == 1 && attackphase != 1 && holdphase != 1) { holdcount = 0; releasephase = 0; attackphase = 1; }
    if (attackphase == 1) { amplitude += (1 * attack); output = input * amplitude; }
    if (amplitude >= 1) { amplitude = 1; attackphase = 0; holdphase = 1; }
    if (holdcount < holdtime && holdphase == 1) { output = input; holdcount++; }
    if (holdcount == holdtime && trigger == 1) { output = input; }
    if (holdcount == holdtime && trigger != 1) { holdphase = 0; releasephase = 1; }
    if (releasephase == 1 && amplitude > 0.) { output = input * (amplitude *= release); }
    st[0] = amplitude; st[V] = output; st[2 * V] = (double)holdcount;
    st[3 * V] = (double)(attackphase | decayphase << 1 | sustainphase << 2 | holdphase << 3 | releasephase << 4);
    return output;
}

/* maxiTrigger::onZX, src/maximilian.h:564-585 */
static double p_on_zx(double* previousValue, double* firstTrigger, double input) {
    double isZX = 0.0;
    if ((*previousValue <= 0.0 || *firstTrigger != 0.0) && input > 0) isZX = 1.0;
    *previousValue = input; *firstTrigger = 0;
    return isZX;
}

/* maxiEnvGen::play, src/maximilian.h:2276-2357; the per-stage counter / currentlevel of the reference are zero for every
 * stage but the current one, so one pair per voice carries them */
static double p_envgen(const eg_shape_t* e, double* st, size_t V, double trigger) {
    double envval = st[0]; size_t phase = (size_t)st[V]; int state = (int)st[2 * V]; int nxc = st[3 * V] != 0.0;
    size_t counter = (size_t)st[4 * V]; double currentlevel = st[5 * V];
    const size_t nst = (size_t)e->n;
    int run = 1;
#define P_RESET() do { counter = 0; currentlevel = 0; phase = 0; state = 1; } while (0)
    if (state == 0) {
        if (p_on_zx(&st[6 * V], &st[7 * V], trigger)) { if (nst > 0) { state = 1; nxc = 0; } else run = 0; }
        else run = 0;
    }
    if (run && state == 1) {
        const eg_stage_t* cs = &e->seg[phase < nst ? phase : 0];
        if (p_on_zx(&st[8 * V], &st[9 * V], -trigger)) nxc = 1;
        if (cs->hold) state = 2;
        else {
            double val = pow(currentlevel, cs->curve);
            val = (1.0 < val) ? 1.0 : val;                           /* maxiMap::linlin, src/maximilian.h:801-805: std::min, then */
            val = (val < 0.0) ? 0.0 : val;                           /* std::max -- a NaN passes both, as it does there */
            envval = ((val - 0.0) / (1.0 - 0.0) * (cs->endlevel - cs->startlevel)) + cs->startlevel;
            counter++;
            if (counter == cs->length) { counter = 0; currentlevel = 0; phase++; }
            else currentlevel += cs->gradient;
            if (e->retrigger) { if (p_on_zx(&st[10 * V], &st[11 * V], trigger)) { nxc = 0; P_RESET(); } }
            run = 0;
        }
    }
    if (run && state == 2) {
        if (p_on_zx(&st[8 * V], &st[9 * V], -trigger)) nxc = 1;
        if (nxc) { state = 1; phase++; }
        if (e->retrigger) { if (p_on_zx(&st[10 * V], &st[11 * V], trigger)) { nxc = 0; P_RESET(); } }
    }
    if (phase == nst) { P_RESET(); if (!e->loop) state = 0; }
#undef P_RESET
    st[0] = envval; st[V] = (double)phase; st[2 * V] = (double)state; st[3 * V] = nxc ? 1.0 : 0.0; st[4 * V] = (double)counter; st[5 * V] = currentlevel;
    return envval;
}

/* maxiBiquad::set for one voice (the expressions of biquad_set above, src/maximilian.h:1375-1479) */
static void p_biquad_set(int type, double cutoff, double Q, double peakGain, double sr, double* cf) {
    bank_t b; double c0, c1, c2, c3, c4; double pc = cutoff, pq = Q, pg = peakGain;
    memset(&b, 0, sizeof(b));
    b.chain.sample_rate = (int32_t)sr; b.chain.biquad_type = type;
    b.p[MXO_P_CUTOFF] = &pc; b.p[MXO_P_RESONANCE] = &pq; b.p[MXO_P_GAIN] = &pg;
    b.cf[0] = &c0; b.cf[1] = &c1; b.cf[2] = &c2; b.cf[3] = &c3; b.cf[4] = &c4;
    biquad_set(&b, 0);
    cf[0] = c0; cf[1] = c1; cf[2] = c2; cf[3] = c3; cf[4] = c4;
}

int32_t mxo_patch_process(void* h, int32_t nframes, const double* const* inputs, double* out, double* mix) {
    patch_t* p = (patch_t*)h;
    if (!p || nframes < 0) return -1;
    const size_t V = (size_t)p->d.voices;
    const double sr = (double)(size_t)p->d.sample_rate;
    const int taps = p->d.delay_taps;
    for (int t = 0; t < nframes; ++t) {
        double m0 = 0.0, m1 = 0.0;
        for (size_t v = 0; v < V; ++v) {
            double* reg = p->reg;
            for (int i = 0; i < 16; ++i) reg[i] = 0.0;          /* registers read 0 until a stage of this sample writes them */
#define FETCH(s) ((s) < 0 ? 0.0 : ((s) >> 8) == 0 ? reg[(s) & 0xff] : ((s) >> 8) == 1 ? p->params[(size_t)((s) & 0xff) * V + v] : \
                  ((s) >> 8) == 2 ? p->consts[(s) & 0xff] : inputs[(s) & 0xff][(size_t)t * V + v])
            for (int si = 0; si < p->d.n_stages; ++si) {
                const mxo_stage* g = &p->stages[si];
                double* st = p->state + (size_t)p->sbase[si] * V + v;      /* slot k at st[k * V] */
                double y = 0.0;
                switch (g->op) {
                    case MXO_OP_OSC: {
                        const double f = FETCH(g->src[0]);
                        if (g->kind >= MXO_OSC_SINEBUF) y = p_osc_table(g->kind, &st[0], &st[V], f, sr);
                        else y = osc_tick(g->kind, &st[0], &st[V], f, FETCH(g->src[1]), sr, FETCH(g->src[1]), FETCH(g->src[2]));
                        break;
                    }
                    case MXO_OP_ENV_ADSR:
                        y = p_env_adsr(st, V, FETCH(g->src[0]), (int)FETCH(g->src[1]), FETCH(g->src[2]), FETCH(g->src[3]), FETCH(g->src[4]),
                                       FETCH(g->src[5]), (long)FETCH(g->src[6]));
                        break;
                    case MXO_OP_ENV_AR:
                        y = p_env_ar(st, V, FETCH(g->src[0]), (int)FETCH(g->src[1]), FETCH(g->src[2]), FETCH(g->src[3]), (long)FETCH(g->src[4]));
                        break;
                    case MXO_OP_ENVGEN: y = p_envgen(&p->eg[g->kind], st, V, FETCH(g->src[0])); break;
                    case MXO_OP_FILTER: {
                        const double input = FETCH(g->src[0]);
                        if (g->kind == MXO_FILT_LORES || g->kind == MXO_FILT_HIRES) {
                            /* maxiFilter::lores / hires, src/maximilian.cpp:455-468 / 471-484 */
                            double cutoff = FETCH(g->src[1]), resonance = FETCH(g->src[2]);
                            double fx = st[0], fy = st[V];
                            if (cutoff < 10) cutoff = 10;
                            if (cutoff > sr) cutoff = sr;
                            if (resonance < 1.) resonance = 1.;
                            double z = cos(MAXI_TWOPI * cutoff / sr);
                            double cc = 2 - 2 * z;
                            double r = (sqrt(2.0) * sqrt(-pow((z - 1.0), 3.0)) + resonance * (z - 1)) / (resonance * (z - 1));
                            fx = fx + (input - fy) * cc;
                            fy = fy + fx;
                            fx = fx * r;
                            st[0] = fx; st[V] = fy;
                            y = g->kind == MXO_FILT_LORES ? fy : input - fy;
                        } else if (g->kind == MXO_FILT_LOPASS) {       /* src/maximilian.cpp:442-446 (outputs[0] defined as 0 initially) */
                            const double cutoff = FETCH(g->src[1]);
                            y = st[0] + cutoff * (input - st[0]);
                            st[0] = y;
                        } else if (g->kind == MXO_FILT_HIPASS) {       /* :449-453 */
                            const double cutoff = FETCH(g->src[1]);
                            y = input - (st[0] + cutoff * (input - st[0]));
                            st[0] = y;
                        } else {                                        /* bandpass, :487-500 */
                            double cutoff = FETCH(g->src[1]), resonance = FETCH(g->src[2]);
                            if (cutoff > (sr * 0.5)) cutoff = (sr * 0.5);
                            if (resonance >= 1.) resonance = 0.999999;
                            double z = cos(MAXI_TWOPI * cutoff / sr);
                            double i0 = (1 - resonance) * (sqrt(resonance * (resonance - 4.0 * pow(z, 2.0) + 2.0) + 1));
                            double i1 = 2 * z * resonance;
                            double i2 = pow((resonance * -1), 2);
                            y = i0 * input + i1 * st[0] + i2 * st[V];
                            st[V] = st[0];
                            st[0] = y;
                        }
                        break;
                    }
                    case MXO_OP_SVF: {
                        /* maxiSVF::setCutoff + setResonance (setParams, src/maximilian.h:1322-1334) then play (:1305-1319) */
                        const double w = FETCH(g->src[0]), freq = FETCH(g->src[1]), res = FETCH(g->src[2]);
                        const double gg = tan(MAXI_PI * freq / sr);
                        const double k = res == 0 ? 0 : 1.0 / res;
                        const double ginv = gg / (1.0 + gg * (gg + k));
                        const double g1 = ginv, g2 = 2.0 * (gg + k) * ginv, g3 = gg * ginv, g4 = 2.0 * ginv;
                        double v0z = st[0], v1 = st[V], v2 = st[2 * V];
                        double v1z = v1, v2z = v2;
                        double v3 = w + v0z - 2.0 * v2z;
                        v1 += g1 * v3 - g2 * v1z;
                        v2 += g3 * v3 + g4 * v1z;
                        v0z = w;
                        const double low = v2, band = v1, high = w - k * v1 - v2, notch = w - k * v1;
                        st[0] = v0z; st[V] = v1; st[2 * V] = v2;
                        y = (low * FETCH(g->src[3])) + (band * FETCH(g->src[4])) + (high * FETCH(g->src[5])) + (notch * FETCH(g->src[6]));
                        break;
                    }
                    case MXO_OP_BIQUAD: {
                        double cf[5];
                        p_biquad_set(g->kind, FETCH(g->src[1]), FETCH(g->src[2]), FETCH(g->src[3]), sr, cf);
                        const double x = FETCH(g->src[0]);
                        double v1 = st[0], v2 = st[V];
                        double v0 = x - (cf[3] * v1) - (cf[4] * v2);
                        y = (cf[0] * v0) + (cf[1] * v1) + (cf[2] * v2);
                        st[V] = v1; st[0] = v0;
                        break;
                    }
                    case MXO_OP_DCBLOCK: {          /* maxiDCBlocker::play, src/maximilian.h:1261-1266 */
                        const double input = FETCH(g->src[0]), R = FETCH(g->src[1]);
                        double ym1 = input - st[0] + R * st[V];
                        st[V] = ym1; st[0] = input;
                        y = ym1;
                        break;
                    }
                    case MXO_OP_NONLIN: {           /* maxiNonlinearity, src/maximilian.h:1076-1137 */
                        double x = FETCH(g->src[0]);
                        const double p1 = FETCH(g->src[1]), p2 = FETCH(g->src[2]);
                        switch (g->kind) {
                            case MXO_NL_ATANDIST: x = (1.0 / atan(p1)) * atan(x * p1); break;
                            case MXO_NL_FASTATANDIST: x = (1.0 / (p1 / (1.0 + 0.28 * (p1 * p1)))) * ((x * p1) / (1.0 + 0.28 * ((x * p1) * (x * p1)))); break;
                            case MXO_NL_SOFTCLIP: if (x >= 1) x = 1; else if (x <= -1) x = -1; else x = (2 / 3.0) * (x - pow(x, 3) / 3.0); break;
                            case MXO_NL_HARDCLIP: x = x >= 1 ? 1 : (x <= -1 ? -1 : x); break;
                            case MXO_NL_ASYMCLIP: if (x >= 1) x = 1; else if (x <= -1) x = -1; else if (x < 0) x = -(pow(-x, p1)); else x = pow(x, p2); break;
                            default: x = (x / (1.0 + 0.28 * (x * x))); break;
                        }
                        y = x;
                        break;
                    }
                    case MXO_OP_DELAY:
                    case MXO_OP_FLANGER: {
                        double* memory = p->rings + ((size_t)p->ringof[si] * V + v) * (size_t)taps;
                        const double input = FETCH(g->src[0]);
                        int size; double feedback;
                        if (g->op == MXO_OP_DELAY) { size = (int)FETCH(g->src[1]); feedback = FETCH(g->src[2]); }
                        else {
                            /* maxiFlanger::flange, src/maximilian.h:1167-1175 */
                            const unsigned int delay = (unsigned int)FETCH(g->src[1]);
                            feedback = FETCH(g->src[2]);
                            const double speed = FETCH(g->src[3]), depth = FETCH(g->src[4]);
                            double lfoVal = osc_tick(MXO_OSC_TRIANGLE, &st[V], &st[2 * V], speed, 0.0, sr, 0.0, 0.0);
                            size = (int)(delay + (lfoVal * depth * delay) + 1);
                        }
                        int phase = (int)st[0];
                        if (phase >= size) phase = 0;                     /* maxiDelayline::dl, src/maximilian.cpp:420-429 */
                        if (phase < 0 || phase >= taps) return -4;
                        double output;
                        if (g->op == MXO_OP_DELAY && g->kind == 1) {      /* dlFromPosition, :431-439 */
                            int position = (int)FETCH(g->src[3]);
                            if (position >= size) position = 0;
                            if (position < 0 || position >= taps) return -4;
                            output = memory[position];
                            memory[phase] = (memory[phase] * feedback) + (input * feedback) * 1.0f;
                        } else {
                            output = memory[phase];
                            memory[phase] = (memory[phase] * feedback) + (input * feedback) * 0.5;
                        }
                        phase += 1;
                        st[0] = (double)phase;
                        if (g->op == MXO_OP_FLANGER) {
                            double normalise = (1 - fabs(output));
                            output *= normalise;
                            y = (output + input) / 2.0;
                        } else y = output;
                        break;
                    }
                    case MXO_OP_CHORUS: {           /* maxiChorus::chorus, src/maximilian.h:1200-1212; slots: dl.phase, dl2.phase, lopass.x, lopass.y */
                        const double input = FETCH(g->src[0]);
                        const unsigned int delay = (unsigned int)FETCH(g->src[1]);
                        const double feedback = FETCH(g->src[2]), speed = FETCH(g->src[3]), depth = FETCH(g->src[4]);
                        double lfoVal = FETCH(g->src[5]);                 /* lfo.noise() */
                        {   /* lopass.lores(lfoVal, speed, 1.0), src/maximilian.cpp:455-468 */
                            double cutoff = speed, resonance = 1.0;
                            double fx = st[2 * V], fy = st[3 * V];
                            if (cutoff < 10) cutoff = 10;
                            if (cutoff > sr) cutoff = sr;
                            if (resonance < 1.) resonance = 1.;
                            double z = cos(MAXI_TWOPI * cutoff / sr);
                            double cc = 2 - 2 * z;
                            double r = (sqrt(2.0) * sqrt(-pow((z - 1.0), 3.0)) + resonance * (z - 1)) / (resonance * (z - 1));
                            fx = fx + (lfoVal - fy) * cc;
                            fy = fy + fx;
                            fx = fx * r;
                            st[2 * V] = fx; st[3 * V] = fy;
                            lfoVal = fy * 2.0;
                        }
                        double outs[2];
                        for (int k = 0; k < 2; ++k) {                     /* dl.dl(input, size, feedback) / dl2.dl(...), src/maximilian.cpp:420-429 */
                            double* memory = p->rings + ((size_t)(p->ringof[si] + k) * V + v) * (size_t)taps;
                            const int size = k == 0 ? (int)(delay + (lfoVal * depth * delay) + 1) : (int)((delay + (lfoVal * depth * delay * 1.02) + 1) * 0.98);
                            const double fbk = k == 0 ? feedback : feedback * 0.99;
                            int phase = (int)st[(size_t)k * V];
                            if (phase >= size) phase = 0;
                            if (phase < 0 || phase >= taps) return -4;
                            outs[k] = memory[phase];
                            memory[phase] = (memory[phase] * fbk) + (input * fbk) * 0.5;
                            phase += 1;
                            st[(size_t)k * V] = (double)phase;
                        }
                        outs[0] *= (1.0 - fabs(outs[0]));
                        outs[1] *= (1.0 - fabs(outs[1]));
                        y = (outs[0] + outs[1] + input) / 3.0;
                        break;
                    }
                    case MXO_OP_ADD: y = FETCH(g->src[0]) + FETCH(g->src[1]); break;
                    case MXO_OP_SUB: y = FETCH(g->src[0]) - FETCH(g->src[1]); break;
                    case MXO_OP_MUL: y = FETCH(g->src[0]) * FETCH(g->src[1]); break;
                    case MXO_OP_DIV: y = FETCH(g->src[0]) / FETCH(g->src[1]); break;
                    case MXO_OP_MIX_STEREO: {       /* maxiMix::stereo, src/maximilian.cpp:503-509 */
                        const double in = FETCH(g->src[0]);
                        double x = FETCH(g->src[1]);
                        if (x > 1) x = 1;
                        if (x < 0) x = 0;
                        m0 += in * sqrt(1.0 - x); m1 += in * sqrt(x);
                        break;
                    }
                    case MXO_OP_OUT: if (out) out[(size_t)t * V + v] = FETCH(g->src[0]); break;
                    default: return -2;
                }
                if (g->dst >= 0) reg[g->dst] = y;
            }
#undef FETCH
        }
        if (mix) { mix[2 * t] = m0; mix[2 * t + 1] = m1; }
    }
    return 0;
}

/* ==================================================================== FFT */

/* ReverseBits, src/libs/fft.cpp:75-85 (the lazily built gFFTBitTable, :87-112, holds the same values) */
static int reverse_bits(int index, int NumBits) {
    int i, rev;
    for (i = rev = 0; i < NumBits; i++) { rev = (rev << 1) | (index & 1); index >>= 1; }
    return rev;
}
static int bits_needed(int PowerOfTwo) { int i; for (i = 0;; i++) if (PowerOfTwo & (1 << i)) return i; }

/* FFT(), src/libs/fft.cpp:118-211: radix-2 decimation in time, float data, float twiddle recurrence
 * restarted for every block, /N on the inverse. */
static void ref_FFT(int NumSamples, int InverseTransform, const float* RealIn, const float* ImagIn,
                    float* RealOut, float* ImagOut) {
    int NumBits, i, j, k, n, BlockSize, BlockEnd;
    double angle_numerator = 2.0 * FFT_M_PI;
    float tr, ti;
    if (InverseTransform) angle_numerator = -angle_numerator;
    NumBits = bits_needed(NumSamples);
    for (i = 0; i < NumSamples; i++) {
        j = reverse_bits(i, NumBits);
        RealOut[j] = RealIn[i];
        ImagOut[j] = (ImagIn == NULL) ? 0.0 : ImagIn[i];
    }
    BlockEnd = 1;
    for (BlockSize = 2; BlockSize <= NumSamples; BlockSize <<= 1) {
        double delta_angle = angle_numerator / (double)BlockSize;
        float sm2 = sin(-2 * delta_angle);
        float sm1 = sin(-delta_angle);
        float cm2 = cos(-2 * delta_angle);
        float cm1 = cos(-delta_angle);
        float w = 2 * cm1;
        float ar0, ar1, ar2, ai0, ai1, ai2;
        for (i = 0; i < NumSamples; i += BlockSize) {
            ar2 = cm2; ar1 = cm1;
            ai2 = sm2; ai1 = sm1;
            for (j = i, n = 0; n < BlockEnd; j++, n++) {
                ar0 = w * ar1 - ar2; ar2 = ar1; ar1 = ar0;
                ai0 = w * ai1 - ai2; ai2 = ai1; ai1 = ai0;
                k = j + BlockEnd;
                tr = ar0 * RealOut[k] - ai0 * ImagOut[k];
                ti = ar0 * ImagOut[k] + ai0 * RealOut[k];
                RealOut[k] = RealOut[j] - tr;
                ImagOut[k] = ImagOut[j] - ti;
                RealOut[j] += tr;
                ImagOut[j] += ti;
            }
        }
        BlockEnd = BlockSize;
    }
    if (InverseTransform) {
        float denom = (float)NumSamples;
        for (i = 0; i < NumSamples; i++) { RealOut[i] /= denom; ImagOut[i] /= denom; }
    }
}

/* RealFFT(), src/libs/fft.cpp:228-282. The double literals (0.5, -2.0, 1.0) promote their
 * sub-expressions to double before the result narrows back to float; kept as written. */
static void ref_RealFFT(int NumSamples, const float* RealIn, float* RealOut, float* ImagOut, float* tmpReal, float* tmpImag) {
    int Half = NumSamples / 2;
    int i;
    float theta = FFT_M_PI / Half;
    for (i = 0; i < Half; i++) { tmpReal[i] = RealIn[2 * i]; tmpImag[i] = RealIn[2 * i + 1]; }
    ref_FFT(Half, 0, tmpReal, tmpImag, RealOut, ImagOut);
    float wtemp = (float)(sin(0.5 * theta));
    float wpr = -2.0 * wtemp * wtemp;
    float wpi = (float)(sin(theta));
    float wr = 1.0 + wpr;
    float wi = wpi;
    int i3;
    float h1r, h1i, h2r, h2i;
    for (i = 1; i < Half / 2; i++) {
        i3 = Half - i;
        h1r = 0.5 * (RealOut[i] + RealOut[i3]);
        h1i = 0.5 * (ImagOut[i] - ImagOut[i3]);
        h2r = 0.5 * (ImagOut[i] + ImagOut[i3]);
        h2i = -0.5 * (RealOut[i] - RealOut[i3]);
        RealOut[i] = h1r + wr * h2r - wi * h2i;
        ImagOut[i] = h1i + wr * h2i + wi * h2r;
        RealOut[i3] = h1r - wr * h2r + wi * h2i;
        ImagOut[i3] = -h1i + wr * h2i + wi * h2r;
        wtemp = wr;
        wr = wtemp * wpr - wi * wpi + wr;
        wi = wi * wpr + wtemp * wpi + wi;
    }
    h1r = RealOut[0];
    RealOut[0] = h1r + ImagOut[0];
    ImagOut[0] = h1r - ImagOut[0];
}

/* fft::genWindow(3, ...), src/libs/fft.cpp:409-413 (Hann, computed in double, stored as float) */
static void gen_hann(int NumSamples, float* window) {
    for (int i = 0; i < NumSamples; i++) window[i] = 0.50 - 0.50 * cos(2 * FFT_M_PI * i / (NumSamples - 1));
}

typedef struct {
    int C, n, hop, bins;
    int* pos;                       /* maxiFFT::pos per channel */
    float* buffer;                  /* [C][n]   maxiFFT::buffer */
    float* window;                  /* [n] */
    float *in_real, *out_real, *out_img, *tmpR, *tmpI;   /* fft::in_real ... (scratch, one channel at a time) */
} stft_t;

/* maxiFFT::setup, src/libs/maxiFFT.cpp:45-60 (windowSize == fftSize, see SURVEY.md A10) */
void* mxo_stft_create(int32_t channels, int32_t fft_size, int32_t hop_size) {
    if (channels <= 0 || fft_size < 4 || (fft_size & (fft_size - 1)) || hop_size <= 0 || hop_size > fft_size) return NULL;
    stft_t* s = (stft_t*)calloc(1, sizeof(stft_t));
    s->C = channels; s->n = fft_size; s->hop = hop_size; s->bins = fft_size / 2;
    s->pos = (int*)malloc(sizeof(int) * (size_t)channels);
    for (int c = 0; c < channels; ++c) s->pos[c] = fft_size - hop_size;
    s->buffer = (float*)calloc((size_t)channels * (size_t)fft_size, sizeof(float));
    s->window = (float*)calloc((size_t)fft_size, sizeof(float));
    gen_hann(fft_size, s->window);
    s->in_real = (float*)calloc((size_t)fft_size, sizeof(float));
    s->out_real = (float*)calloc((size_t)fft_size, sizeof(float));
    s->out_img = (float*)calloc((size_t)fft_size, sizeof(float));
    s->tmpR = (float*)calloc((size_t)fft_size, sizeof(float));
    s->tmpI = (float*)calloc((size_t)fft_size, sizeof(float));
    return s;
}
void mxo_stft_destroy(void* h) {
    stft_t* s = (stft_t*)h; if (!s) return;
    free(s->pos); free(s->buffer); free(s->window); free(s->in_real); free(s->out_real); free(s->out_img);
    free(s->tmpR); free(s->tmpI); free(s);
}
int32_t mxo_stft_window(void* h, float* w) {
    stft_t* s = (stft_t*)h; if (!s || !w) return -1;
    memcpy(w, s->window, sizeof(float) * (size_t)s->n); return 0;
}

/* maxiFFT::process, src/libs/maxiFFT.cpp:65-91 -> fft::powerSpectrum, src/libs/fft.cpp:519-524
 * = calcFFT :499-505 + cartToPol :507-515 (sqrt/atan2 on floats are the float overloads, SURVEY.md A17) */
int32_t mxo_stft_process(void* h, const float* in, int32_t n, int32_t max_frames,
                         float* mags, float* phases, float* re, float* im) {
    stft_t* s = (stft_t*)h;
    if (!s || !in || n < 0) return -1;
    int frames = 0;
    for (int c = 0; c < s->C; ++c) {
        float* buffer = s->buffer + (size_t)c * (size_t)s->n;
        int pos = s->pos[c];
        int k = 0;
        for (int t = 0; t < n; ++t) {
            buffer[pos++] = in[(size_t)c * (size_t)n + (size_t)t];
            if (pos == s->n) {
                if (k >= max_frames) return -3;
                for (int i = 0; i < s->n; i++) s->in_real[i] = buffer[i] * s->window[i];
                ref_RealFFT(s->n, s->in_real, s->out_real, s->out_img, s->tmpR, s->tmpI);
                size_t o = ((size_t)c * (size_t)max_frames + (size_t)k) * (size_t)s->bins;
                for (int i = 0; i < s->bins; i++) {
                    float power = s->out_real[i] * s->out_real[i] + s->out_img[i] * s->out_img[i];
                    if (mags) mags[o + i] = sqrtf(power);
                    if (phases) phases[o + i] = atan2f(s->out_img[i], s->out_real[i]);
                    if (re) re[o + i] = s->out_real[i];
                    if (im) im[o + i] = s->out_img[i];
                }
                memmove(buffer, buffer + s->hop, sizeof(float) * (size_t)(s->n - s->hop));
                pos = s->n - s->hop;
                ++k;
            }
        }
        s->pos[c] = pos;
        frames = k;
    }
    return frames;
}

/* fft::convToDB (src/libs/fft.cpp:526-534), maxiFFT::spectralFlatness / spectralCentroid (src/libs/maxiFFT.cpp:113-132).
 * The unqualified log10 / fabs on floats are the float overloads in the reference (SURVEY.md A17); sums are float, in bin order. */
int32_t mxo_spectral_features(const float* mags, int32_t n_frames, int32_t fft_size, int32_t sample_rate,
                              float* db, float* flatness, float* centroid) {
    if (!mags || n_frames < 0 || fft_size < 4 || (fft_size & (fft_size - 1))) return -1;
    const int bins = fft_size / 2;
    for (int fr = 0; fr < n_frames; ++fr) {
        const float* magnitudes = mags + (size_t)fr * (size_t)bins;
        if (db) {
            float* out = db + (size_t)fr * (size_t)bins;
            for (int i = 0; i < bins; i++) {
                if (magnitudes[i] < 0.000001) out[i] = 0;
                else out[i] = 20.0 * log10f(magnitudes[i] + 1);
            }
        }
        if (flatness) {
            float geometricMean = 0, arithmaticMean = 0;
            for (size_t i = 0; i < (size_t)bins; i++) {
                if (magnitudes[i] != 0) geometricMean += logf(magnitudes[i]);
                arithmaticMean += magnitudes[i];
            }
            geometricMean = expf(geometricMean / (float)bins);
            arithmaticMean /= (float)bins;
            flatness[fr] = arithmaticMean != 0 ? geometricMean / arithmaticMean : 0;
        }
        if (centroid) {
            float x = 0, y = 0;
            for (size_t i = 0; i < (size_t)bins; i++) {
                x += fabsf(magnitudes[i]) * i;
                y += fabsf(magnitudes[i]);
            }
            centroid[fr] = y != 0 ? x / y * ((float)(size_t)sample_rate / fft_size) : 0;
        }
    }
    return 0;
}

/* ======================================================= spectral analysers */

typedef struct { int C, nSpectrum, nAverages; int* spe2avg; float *averages, *peaks; int* peakHoldTimes;
                 int peakHoldTime; float peakDecayRate, linearEQIntercept, linearEQSlope; } octave_t;

/* maxiFFTOctaveAnalyzer::setup, src/libs/maxiFFT.cpp:201-262 (float arithmetic throughout; pow on floats is powf there) */
void* mxo_octave_create(int32_t channels, float samplingRate, int32_t nBandsInTheFFT, int32_t nAveragesPerOctave) {
    if (channels <= 0 || nBandsInTheFFT <= 0) return NULL;
    octave_t* o = (octave_t*)calloc(1, sizeof(octave_t));
    o->C = channels; o->nSpectrum = nBandsInTheFFT;
    float spectrumFrequencySpan = (samplingRate / 2.0f) / (float)(o->nSpectrum);
    if (nAveragesPerOctave == 0) nAveragesPerOctave = 1;
    float averageFrequencyIncrement = powf(2.0f, 1.0f / (float)(nAveragesPerOctave));
    float firstOctaveFrequency = 55.0f;
    o->spe2avg = (int*)calloc((size_t)o->nSpectrum, sizeof(int));
    int avgidx = 0;
    float averageFreq = firstOctaveFrequency;
    float spectrumFreq = spectrumFrequencySpan;
    for (int speidx = 0; speidx < o->nSpectrum; speidx++) {
        while (spectrumFreq > averageFreq) { avgidx++; averageFreq *= averageFrequencyIncrement; }
        o->spe2avg[speidx] = avgidx;
        spectrumFreq += spectrumFrequencySpan;
    }
    o->nAverages = avgidx;
    o->averages = (float*)calloc((size_t)channels * (size_t)(avgidx ? avgidx : 1), sizeof(float));
    o->peaks = (float*)calloc((size_t)channels * (size_t)(avgidx ? avgidx : 1), sizeof(float));
    o->peakHoldTimes = (int*)calloc((size_t)channels * (size_t)(avgidx ? avgidx : 1), sizeof(int));
    o->peakHoldTime = 0; o->peakDecayRate = 0.9f; o->linearEQIntercept = 1.0f; o->linearEQSlope = 0.0f;
    return o;
}
void mxo_octave_destroy(void* h) { octave_t* o = (octave_t*)h; if (!o) return; free(o->spe2avg); free(o->averages); free(o->peaks); free(o->peakHoldTimes); free(o); }
int32_t mxo_octave_n_averages(void* h) { return h ? ((octave_t*)h)->nAverages : -1; }
int32_t mxo_octave_config(void* h, int32_t hold, float decay, float intercept, float slope) {
    octave_t* o = (octave_t*)h; if (!o) return -1;
    o->peakHoldTime = hold; o->peakDecayRate = decay; o->linearEQIntercept = intercept; o->linearEQSlope = slope;
    return 0;
}
/* maxiFFTOctaveAnalyzer::calculate, src/libs/maxiFFT.cpp:264-300 */
int32_t mxo_octave_process(void* h, const float* mags, int32_t frames, float* avg_out, float* peak_out) {
    octave_t* o = (octave_t*)h;
    if (!o || !mags || frames < 0) return -1;
    const int nA = o->nAverages;
    for (int c = 0; c < o->C; ++c) {
        float* averages = o->averages + (size_t)c * nA; float* peaks = o->peaks + (size_t)c * nA; int* peakHoldTimes = o->peakHoldTimes + (size_t)c * nA;
        for (int f = 0; f < frames; ++f) {
            const float* fftData = mags + ((size_t)c * frames + f) * (size_t)o->nSpectrum;
            int last_avgidx = 0;
            float sum = 0.0f;
            int count = 0;
            for (int speidx = 0; speidx < o->nSpectrum; speidx++) {
                count++;
                sum += fftData[speidx] * (o->linearEQIntercept + (float)(speidx)*o->linearEQSlope);
                int avgidx = o->spe2avg[speidx];
                if (avgidx != last_avgidx) {
                    for (int j = last_avgidx; j < avgidx; j++) averages[j] = sum / (float)(count);
                    count = 0;
                    sum = 0.0f;
                }
                last_avgidx = avgidx;
            }
            if ((count > 0) && (last_avgidx < nA)) averages[last_avgidx] = sum / (float)(count);
            for (int i = 0; i < nA; i++) {
                if (averages[i] >= peaks[i]) { peaks[i] = averages[i]; peakHoldTimes[i] = o->peakHoldTime; }
                else { if (peakHoldTimes[i] > 0) peakHoldTimes[i]--; else peaks[i] *= o->peakDecayRate; }
            }
            if (avg_out) memcpy(avg_out + ((size_t)c * frames + f) * nA, averages, sizeof(float) * (size_t)nA);
            if (peak_out) memcpy(peak_out + ((size_t)c * frames + f) * nA, peaks, sizeof(float) * (size_t)nA);
        }
    }
    return 0;
}

/* maxiBarkScaleAnalyser, src/libs/maxiBark.h:25-126. binToHz is UNSIGNED INTEGER arithmetic (bin*sR/bS) returned as a double;
 * currentBandEnd is an int; bbLimits has 24 slots and setup() writes bbLimits[24] (the member behind it): 25 slots here. */
int32_t mxo_bark(const float* spectrum, int32_t n_frames, int32_t sample_rate, int32_t buffer_size, double* specific_out, double* relative_out, double* total_out) {
    if (!spectrum || n_frames < 0 || buffer_size < 4 || buffer_size / 2 > 2048) return -1;
    const unsigned int sR = (unsigned int)sample_rate, bS = (unsigned int)buffer_size, specSize = bS / 2;
    const int NUM_BARK_BANDS = 24;
    static double barkScale[2048];
    int bbLimits[32];
    memset(bbLimits, 0, sizeof(bbLimits));
    for (unsigned int i = 0; i < specSize; i++) {
        double hz = (double)(i * sR / bS);
        barkScale[i] = 13.0 * atan(hz / 1315.8) + 3.5 * atan(pow((hz / 7518.0), 2));
    }
    bbLimits[0] = 0;
    int currentBandEnd = barkScale[specSize - 1] / NUM_BARK_BANDS;
    int currentBand = 1;
    for (unsigned int i = 0; i < specSize; i++) {
        while (barkScale[i] > currentBandEnd) {
            if (currentBand < 32) bbLimits[currentBand] = (int)i;
            currentBand++;
            currentBandEnd = currentBand * barkScale[specSize - 1] / NUM_BARK_BANDS;
        }
    }
    bbLimits[NUM_BARK_BANDS] = (int)specSize - 1;
    for (int f = 0; f < n_frames; ++f) {
        const float* normalisedSpectrum = spectrum + (size_t)f * specSize;
        double specific[24];
        for (int i = 0; i < NUM_BARK_BANDS; i++) {
            double sum = 0;
            for (int j = bbLimits[i]; j < bbLimits[i + 1]; j++) sum += normalisedSpectrum[j];
            specific[i] = pow(sum, 0.23);
        }
        double max = 0;
        for (int i = 0; i < NUM_BARK_BANDS; i++) if (specific[i] > max) max = specific[i];
        double total = 0;
        for (int i = 0; i < 24; i++) total += specific[i];
        for (int i = 0; i < NUM_BARK_BANDS; i++) {
            if (specific_out) specific_out[(size_t)f * 24 + i] = specific[i];
            if (relative_out) relative_out[(size_t)f * 24 + i] = specific[i] / max;
        }
        if (total_out) total_out[f] = total;
    }
    return 0;
}

/* =================================================================== MFCC */

typedef struct {
    unsigned numBins, numFilters, numCoeffs;
    double* melFilters;   /* idx = filter + bin*numFilters, src/libs/maxiMFCC.h:157 */
    double* dctMatrix;    /* idx = i + j*numCoeffs,        src/libs/maxiMFCC.h:194 */
    double* melBands;
} mfcc_t;

static double hzToMel(double hz) { return 2595.0 * (log10(hz / 700.0 + 1.0)); }        /* maxiMFCC.h:30-32 */
static double melToHz(double mel) { return 700.0 * (pow(10, mel / 2595.0) - 1.0); }    /* maxiMFCC.h:36-38 */

/* maxiMFCCAnalyser<double>::setup :56-75, calcMelFilterBank :118-182, createDCTCoeffs :183-203 */
void* mxo_mfcc_create(int32_t num_bins, int32_t num_filters, int32_t num_coeffs,
                      double minFreq, double maxFreq, int32_t sample_rate) {
    if (num_bins <= 0 || num_filters <= 0 || num_coeffs <= 0) return NULL;
    mfcc_t* m = (mfcc_t*)calloc(1, sizeof(mfcc_t));
    const unsigned numBins = (unsigned)num_bins, numFilters = (unsigned)num_filters, numCoeffs = (unsigned)num_coeffs;
    m->numBins = numBins; m->numFilters = numFilters; m->numCoeffs = numCoeffs;
    m->melBands = (double*)calloc(numFilters, sizeof(double));
    m->dctMatrix = (double*)calloc((size_t)numCoeffs * numFilters, sizeof(double));
    /* column 0 (filter 0) is never written by the reference (loop starts at 1, :149): zero */
    m->melFilters = (double*)calloc((size_t)numFilters * numBins, sizeof(double));
    {
        const double sampleRate = (double)(unsigned)sample_rate;
        double mel, dMel, maxMel, minMel, nyquist, binFreq, start, thisF, nextF, prevF;
        nyquist = sampleRate / 2;
        if (maxFreq > nyquist) maxFreq = nyquist;
        maxMel = hzToMel(maxFreq);
        minMel = hzToMel(minFreq);
        dMel = (maxMel - minMel) / (numFilters + 2 - 1);
        double* filtPos = (double*)malloc(sizeof(double) * (numFilters + 2));
        mel = minMel;
        for (unsigned i = 0; i < numFilters + 2; i++) { filtPos[i] = melToHz(mel); mel += dMel; }
        for (unsigned filter = 1; filter < numFilters; filter++) {
            for (unsigned bin = 0; bin < numBins; bin++) {
                binFreq = (double)sampleRate / (double)(int)numBins * (double)(int)bin;   /* sr/numBins, not sr/fftSize: SURVEY.md A13 */
                thisF = filtPos[filter]; nextF = filtPos[filter + 1]; prevF = filtPos[filter - 1];
                size_t idx = filter + ((size_t)bin * numFilters);
                if (binFreq > nextF || binFreq < prevF) {
                    m->melFilters[idx] = 0;
                } else {
                    double height = 2.0 / (nextF - prevF);
                    if (binFreq < thisF) {
                        start = prevF;
                        m->melFilters[idx] = (binFreq - start) * (height / (thisF - start));
                    } else {
                        m->melFilters[idx] = height + ((binFreq - thisF) * (-height / (nextF - thisF)));
                    }
                }
            }
        }
        free(filtPos);
    }
    {
        double k = 3.14159265358979323846 / numFilters;
        double w1 = 1.0 / (sqrt((double)numFilters));
        double w2 = sqrt(2.0 / numFilters);
        for (unsigned i = 0; i < numCoeffs; i++) {
            for (unsigned j = 0; j < numFilters; j++) {
                size_t idx = i + ((size_t)j * numCoeffs);
                if (i == 0) m->dctMatrix[idx] = w1 * cos(k * (int)(i + 1) * ((int)j + 0.5));
                else m->dctMatrix[idx] = w2 * cos(k * (int)(i + 1) * ((int)j + 0.5));
            }
        }
    }
    return m;
}
void mxo_mfcc_destroy(void* h) { mfcc_t* m = (mfcc_t*)h; if (!m) return; free(m->melFilters); free(m->dctMatrix); free(m->melBands); free(m); }

/* maxiMFCC::mfcc :77-81 = melFilterAndLogSq_Part2 (src/libs/maxiMFCC.cpp:48-66) + dct (maxiMFCC.h:98-111) */
int32_t mxo_mfcc_process(void* h, const float* mags, int32_t n, double* coeffs, double* melbands) {
    mfcc_t* m = (mfcc_t*)h;
    if (!m || !mags || !coeffs) return -1;
    for (int f = 0; f < n; ++f) {
        const float* powerSpectrum = mags + (size_t)f * m->numBins;
        double* mfccs = coeffs + (size_t)f * m->numCoeffs;
        for (unsigned filter = 0; filter < m->numFilters; filter++) {
            m->melBands[filter] = 0.0;
            for (unsigned bin = 0; bin < m->numBins; bin++) {
                size_t idx = filter + ((size_t)bin * m->numFilters);
                m->melBands[filter] += (m->melFilters[idx] * powerSpectrum[bin]);
            }
        }
        for (unsigned filter = 0; filter < m->numFilters; filter++)
            m->melBands[filter] = m->melBands[filter] > 0.000001 ? log(m->melBands[filter] * m->melBands[filter]) : 0.0;
        for (unsigned i = 0; i < m->numCoeffs; i++) mfccs[i] = 0.0;
        for (unsigned i = 0; i < m->numCoeffs; i++)
            for (unsigned j = 0; j < m->numFilters; j++) {
                size_t idx = i + ((size_t)j * m->numCoeffs);
                mfccs[i] += (m->dctMatrix[idx] * m->melBands[j]);
            }
        for (unsigned i = 0; i < m->numCoeffs; i++) mfccs[i] /= m->numCoeffs;
        if (melbands) memcpy(melbands + (size_t)f * m->numFilters, m->melBands, sizeof(double) * m->numFilters);
    }
    return 0;
}

/* ================================================================== ISTFT */

typedef struct {
    int C, n, hop, bins;
    int* pos;
    float* buffer;        /* [C][n] maxiIFFT::buffer */
    float* window;
    float *ifftOut, *in_real, *in_img, *out_real, *out_img;
} istft_t;

/* maxiIFFT::setup, src/libs/maxiFFT.cpp:141-152 */
void* mxo_istft_create(int32_t channels, int32_t fft_size, int32_t hop_size) {
    if (channels <= 0 || fft_size < 4 || (fft_size & (fft_size - 1)) || hop_size <= 0 || hop_size > fft_size) return NULL;
    istft_t* s = (istft_t*)calloc(1, sizeof(istft_t));
    s->C = channels; s->n = fft_size; s->hop = hop_size; s->bins = fft_size / 2;
    s->pos = (int*)calloc((size_t)channels, sizeof(int));
    s->buffer = (float*)calloc((size_t)channels * (size_t)fft_size, sizeof(float));
    s->window = (float*)calloc((size_t)fft_size, sizeof(float));
    gen_hann(fft_size, s->window);
    s->ifftOut = (float*)calloc((size_t)fft_size, sizeof(float));
    s->in_real = (float*)calloc((size_t)fft_size, sizeof(float));
    s->in_img = (float*)calloc((size_t)fft_size, sizeof(float));
    s->out_real = (float*)calloc((size_t)fft_size, sizeof(float));
    s->out_img = (float*)calloc((size_t)fft_size, sizeof(float));
    return s;
}
void mxo_istft_destroy(void* h) {
    istft_t* s = (istft_t*)h; if (!s) return;
    free(s->pos); free(s->buffer); free(s->window); free(s->ifftOut); free(s->in_real); free(s->in_img);
    free(s->out_real); free(s->out_img); free(s);
}

/* maxiIFFT::process (SPECTRUM), src/libs/maxiFFT.cpp:154-192 -> fft::inversePowerSpectrum :621-624
 * = polToCart :590-603 (cosf/sinf) + calcIFFT :605-610 */
int32_t mxo_istft_process(void* h, const float* mags, const float* phases, int32_t frames, float* out) {
    istft_t* s = (istft_t*)h;
    if (!s || !mags || !phases || !out || frames < 0) return -1;
    for (int c = 0; c < s->C; ++c) {
        float* buffer = s->buffer + (size_t)c * (size_t)s->n;
        int pos = s->pos[c];
        for (int f = 0; f < frames; ++f) {
            const float* magnitude = mags + ((size_t)c * (size_t)frames + (size_t)f) * (size_t)s->bins;
            const float* phase = phases + ((size_t)c * (size_t)frames + (size_t)f) * (size_t)s->bins;
            for (int t = 0; t < s->hop; ++t) {
                if (0 == pos) {
                    for (int i = 0; i < s->n; i++) s->ifftOut[i] = 0;
                    for (int i = 0; i < s->bins; i++) {
                        s->in_real[i] = magnitude[i] * cosf(phase[i]);
                        s->in_img[i] = magnitude[i] * sinf(phase[i]);
                    }
                    memset(s->in_real + s->bins, 0, sizeof(float) * (size_t)s->bins);
                    memset(s->in_img + s->bins, 0, sizeof(float) * (size_t)s->bins);
                    ref_FFT(s->n, 1, s->in_real, s->in_img, s->out_real, s->out_img);
                    for (int i = 0; i < s->n; i++) s->ifftOut[i] += s->out_real[i] * s->window[i];
                    memmove(buffer, buffer + s->hop, sizeof(float) * (size_t)(s->n - s->hop));
                    memset(buffer + (s->n - s->hop), 0, sizeof(float) * (size_t)s->hop);
                    for (int i = 0; i < s->n; i++) buffer[i] += s->ifftOut[i];
                }
                out[(size_t)c * (size_t)frames * (size_t)s->hop + (size_t)f * (size_t)s->hop + (size_t)t] = buffer[pos];
                if (s->hop == ++pos) pos = 0;
            }
        }
        s->pos[c] = pos;
    }
    return 0;
}
