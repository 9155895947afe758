/*
 * ref_shim.cpp -- TEST INFRASTRUCTURE ONLY.
 *
 * Drives the UNMODIFIED reference classes (compiled from /root/reference/src by
 * oracle/Makefile, never copied into this repository) behind oracle_api.h.
 * Built into oracle/_ref/libmaxiref.so. This file contains no DSP of its own:
 * every sample comes out of a reference method call.
 *
 * Construction rules (SURVEY.md section 8c): objects live in zero-filled storage
 * (calloc + placement new) because maxiDelayline::phase, every maxiEnv field and
 * maxiFilter::outputs[] are otherwise indeterminate; maxiSettings::setup() runs
 * before any object is built (maxiSVF and maxiMFCC read the rate at construction).
 */
#include <cmath>
#include <cstdlib>
#include <cstring>
#include <new>
#include <vector>
#include <iostream>
#include <algorithm>
#include <numeric>
#include <functional>
#include <string>
#include <map>
#include <valarray>

/* state read-back for the tests needs private members (maxiOsc::phase, maxiDelayline::memory ...):
 * the Makefile passes -fno-access-control, which switches off access checking without
 * touching layout or code generation. */
#include "maximilian.h"
#include "maxiFFT.h"
#include "maxiMFCC.h"
/* maxiBarkScaleAnalyser::setup writes bbLimits[24] of an int[24] (src/libs/maxiBark.h:52-60): undefined behaviour that GCC's
 * loop optimisations turn into a crash at -O2. The class is compiled without optimisation (same arithmetic, IEEE either way);
 * the shim gives the object room behind bbLimits. */
#pragma GCC push_options
#pragma GCC optimize ("O0")
#include "maxiBark.h"
#pragma GCC pop_options

#include "oracle_api.h"

extern double sineBuffer[514];      /* src/maximilian.cpp:63 (external linkage there, not declared in the header) */
extern double transition[1001];     /* src/maximilian.cpp:67 */

namespace {

struct RefVoice {
    maxiOsc osc;
    maxiFilter filt;
    maxiSVF svf;
    maxiBiquad bq;
    maxiEnv env;
    maxiMix mixer;
};

struct RefBank {
    mxo_chain chain;
    int V;
    RefVoice* voices;          /* calloc'ed, placement-constructed */
    maxiDelayline** delays;    /* one 5.6 MB object per voice when delay_on */
    std::vector<double> p[MXO_P_COUNT];
};

template <class T> T* zeroed_new() {
    void* mem = calloc(1, sizeof(T));
    if (!mem) return nullptr;
    return new (mem) T();
}

void apply_svf(RefBank* b) {
    if (b->p[MXO_P_CUTOFF].empty() || b->p[MXO_P_RESONANCE].empty()) return;
    for (int v = 0; v < b->V; ++v) {
        b->voices[v].svf.setCutoff(b->p[MXO_P_CUTOFF][v]);
        b->voices[v].svf.setResonance(b->p[MXO_P_RESONANCE][v]);
    }
}
void apply_biquad(RefBank* b) {
    if (b->p[MXO_P_CUTOFF].empty() || b->p[MXO_P_RESONANCE].empty()) return;
    for (int v = 0; v < b->V; ++v) {
        double g = b->p[MXO_P_GAIN].empty() ? 0.0 : b->p[MXO_P_GAIN][v];
        b->voices[v].bq.set((maxiBiquad::filterTypes)b->chain.biquad_type,
                            b->p[MXO_P_CUTOFF][v], b->p[MXO_P_RESONANCE][v], g);
    }
}

inline double run_osc(maxiOsc& o, int kind, double f, double duty, double pstart, double pend) {
    switch (kind) {
        case MXO_OSC_SINEWAVE: return o.sinewave(f);
        case MXO_OSC_COSWAVE:  return o.coswave(f);
        case MXO_OSC_PHASOR:   return o.phasor(f);
        case MXO_OSC_SAW:      return o.saw(f);
        case MXO_OSC_SQUARE:   return o.square(f);
        case MXO_OSC_PULSE:    return o.pulse(f, duty);
        case MXO_OSC_IMPULSE:  return o.impulse(f);
        case MXO_OSC_TRIANGLE: return o.triangle(f);
        case MXO_OSC_PHASORBETWEEN: return o.phasorBetween(f, pstart, pend);
    }
    return 0.0;
}

}  // namespace

extern "C" {

const char* mxo_kind(void) { return "reference"; }

void* mxo_bank_create(const mxo_chain* chain, int32_t voices) {
    if (!chain || voices <= 0) return nullptr;
    maxiSettings::setup((size_t)chain->sample_rate, 2, 1024);
    RefBank* b = new RefBank();
    b->chain = *chain;
    b->V = voices;
    b->voices = (RefVoice*)calloc((size_t)voices, sizeof(RefVoice));
    for (int v = 0; v < voices; ++v) new (&b->voices[v]) RefVoice();
    b->delays = nullptr;
    if (chain->delay_on) {
        b->delays = (maxiDelayline**)calloc((size_t)voices, sizeof(maxiDelayline*));
        for (int v = 0; v < voices; ++v) {
            b->delays[v] = zeroed_new<maxiDelayline>();
            if (!b->delays[v]) { return nullptr; }
        }
    }
    /* defaults so that an unset parameter behaves like an untouched reference object */
    b->p[MXO_P_FREQ].assign(voices, 0.0);
    b->p[MXO_P_DUTY].assign(voices, 0.5);
    b->p[MXO_P_PHASOR_START].assign(voices, 0.0);
    b->p[MXO_P_PHASOR_END].assign(voices, 1.0);
    b->p[MXO_P_DELAY_SIZE].assign(voices, 1.0);
    b->p[MXO_P_DELAY_FEEDBACK].assign(voices, 0.0);
    b->p[MXO_P_PAN].assign(voices, 0.5);
    b->p[MXO_P_DELAY_POSITION].assign(voices, 0.0);
    b->p[MXO_P_ENV_ATTACK].assign(voices, 0.0);
    b->p[MXO_P_ENV_RELEASE].assign(voices, 0.0);
    b->p[MXO_P_ENV_HOLDTIME].assign(voices, 1.0);
    return b;
}

void mxo_bank_destroy(void* h) {
    RefBank* b = (RefBank*)h;
    if (!b) return;
    if (b->delays) {
        for (int v = 0; v < b->V; ++v) { if (b->delays[v]) { b->delays[v]->~maxiDelayline(); free(b->delays[v]); } }
        free(b->delays);
    }
    for (int v = 0; v < b->V; ++v) b->voices[v].~RefVoice();
    free(b->voices);
    delete b;
}

int32_t mxo_bank_set(void* h, int32_t id, const double* x) {
    RefBank* b = (RefBank*)h;
    if (!b || !x || id < 0 || id >= MXO_P_COUNT) return -1;
    maxiSettings::setup((size_t)b->chain.sample_rate, 2, 1024);
    b->p[id].assign(x, x + b->V);
    switch (id) {
        case MXO_P_PHASE: for (int v = 0; v < b->V; ++v) b->voices[v].osc.phaseReset(x[v]); break;
        case MXO_P_CUTOFF: case MXO_P_RESONANCE: case MXO_P_GAIN:
            if (b->chain.filt_kind == MXO_FILT_SVF) apply_svf(b);
            if (b->chain.filt_kind == MXO_FILT_BIQUAD) apply_biquad(b);
            break;
        case MXO_P_ENV_ATTACK:  for (int v = 0; v < b->V; ++v) b->voices[v].env.attack = x[v]; break;
        case MXO_P_ENV_DECAY:   for (int v = 0; v < b->V; ++v) b->voices[v].env.decay = x[v]; break;
        case MXO_P_ENV_SUSTAIN: for (int v = 0; v < b->V; ++v) b->voices[v].env.setSustain(x[v]); break;
        case MXO_P_ENV_RELEASE: for (int v = 0; v < b->V; ++v) b->voices[v].env.release = x[v]; break;
        case MXO_P_ENV_HOLDTIME:for (int v = 0; v < b->V; ++v) b->voices[v].env.holdtime = (long)x[v]; break;
        default: break;
    }
    return 0;
}

int32_t mxo_bank_get(void* h, int32_t id, double* x) {
    RefBank* b = (RefBank*)h;
    if (!b || !x) return -1;
    const int fk = b->chain.filt_kind;
    for (int v = 0; v < b->V; ++v) {
        RefVoice& r = b->voices[v];
        switch (id) {
            case MXO_P_PHASE: x[v] = r.osc.phase; break;
            case MXO_S_FILT_0: x[v] = fk == MXO_FILT_SVF ? r.svf.v0z : fk == MXO_FILT_BIQUAD ? r.bq.v[1] : r.filt.x; break;
            case MXO_S_FILT_1: x[v] = fk == MXO_FILT_SVF ? r.svf.v1  : fk == MXO_FILT_BIQUAD ? r.bq.v[2] : r.filt.y; break;
            case MXO_S_FILT_2: x[v] = fk == MXO_FILT_SVF ? r.svf.v2 : 0.0; break;
            case MXO_S_ENV_AMPLITUDE: x[v] = r.env.amplitude; break;
            case MXO_S_ENV_OUTPUT: x[v] = r.env.output; break;
            case MXO_S_ENV_HOLDCOUNT: x[v] = (double)r.env.holdcount; break;
            case MXO_S_ENV_FLAGS:
                x[v] = (double)((r.env.attackphase & 1) | (r.env.decayphase & 1) << 1 | (r.env.sustainphase & 1) << 2 |
                                (r.env.holdphase & 1) << 3 | (r.env.releasephase & 1) << 4);
                break;
            case MXO_S_DELAY_PHASE: x[v] = b->delays ? (double)b->delays[v]->phase : 0.0; break;
            case MXO_S_OSC_OUTPUT: x[v] = r.osc.output; break;
            default:
                if (id >= 0 && id < MXO_P_COUNT && !b->p[id].empty()) x[v] = b->p[id][v]; else return -1;
        }
    }
    return 0;
}

int32_t mxo_bank_process(void* h, int32_t nframes, const int32_t* trig_on, const int32_t* trig_off,
                         double* out, double* mix, int32_t first, int32_t count) {
    return mxo_bank_process_fm(h, nframes, nullptr, trig_on, trig_off, out, mix, first, count);
}

int32_t mxo_bank_process_fm(void* h, int32_t nframes, const double* freq_tv, const int32_t* trig_on, const int32_t* trig_off,
                            double* out, double* mix, int32_t first, int32_t count) {
    return mxo_bank_process_mod(h, nframes, freq_tv, nullptr, nullptr, trig_on, trig_off, out, mix, first, count);
}

int32_t mxo_bank_process_mod(void* h, int32_t nframes, const double* freq_tv, const double* cutoff_tv, const double* delay_size_tv,
                             const int32_t* trig_on, const int32_t* trig_off, double* out, double* mix, int32_t first, int32_t count) {
    return mxo_bank_process_mod2(h, nframes, freq_tv, cutoff_tv, delay_size_tv, nullptr, trig_on, trig_off, out, mix, first, count);
}

/* ... and with the envelope's trigger given for every sample: trig_tv[t][v] bytes, maxiEnv::trigger as the patch sets it before each
 * call (src/maximilian.h:913; cpp/commandline/maximilian_examples/10.Filters/main.cpp:27-36) */
int32_t mxo_bank_process_mod2(void* h, int32_t nframes, const double* freq_tv, const double* cutoff_tv, const double* delay_size_tv,
                              const uint8_t* trig_tv, const int32_t* trig_on, const int32_t* trig_off, double* out, double* mix, int32_t first, int32_t count) {
    RefBank* b = (RefBank*)h;
    if (!b || nframes < 0 || first < 0 || count < 0 || first + count > b->V) return -1;
    const mxo_chain& c = b->chain;
    const int V = b->V;
    const double* freq = b->p[MXO_P_FREQ].data();
    const double* duty = b->p[MXO_P_DUTY].data();
    const double* fc = b->p[MXO_P_CUTOFF].empty() ? nullptr : b->p[MXO_P_CUTOFF].data();
    const double* q = b->p[MXO_P_RESONANCE].empty() ? nullptr : b->p[MXO_P_RESONANCE].data();
    const double* dsize = b->p[MXO_P_DELAY_SIZE].data();
    const double* dfb = b->p[MXO_P_DELAY_FEEDBACK].data();
    const double* pan = b->p[MXO_P_PAN].data();
    if ((c.filt_kind == MXO_FILT_LORES || c.filt_kind == MXO_FILT_HIRES) && ((!fc && !cutoff_tv) || !q)) return -2;
    if (cutoff_tv && c.filt_kind == MXO_FILT_BIQUAD) return -3;
    if (delay_size_tv && !c.delay_on) return -3;
    std::vector<double> two(2, 0.0);
    for (int t = 0; t < nframes; ++t) {
        double m0 = 0.0, m1 = 0.0;
        for (int v = first; v < first + count; ++v) {
            RefVoice& r = b->voices[v];
            double x = run_osc(r.osc, c.osc_kind, freq_tv ? freq_tv[(size_t)t * V + v] : freq[v], duty[v],
                               b->p[MXO_P_PHASOR_START][v], b->p[MXO_P_PHASOR_END][v]);
            if (c.env_kind == MXO_ENV_ADSR) {
                int trig = trig_tv ? (int)trig_tv[(size_t)t * (size_t)V + (size_t)v] : (trig_on && trig_off && t >= trig_on[v] && t < trig_off[v]) ? 1 : 0;
                x = r.env.adsr(x, trig);
            } else if (c.env_kind == MXO_ENV_AR) {
                int trig = trig_tv ? (int)trig_tv[(size_t)t * (size_t)V + (size_t)v] : (trig_on && trig_off && t >= trig_on[v] && t < trig_off[v]) ? 1 : 0;
                x = r.env.ar(x, b->p[MXO_P_ENV_ATTACK][v], b->p[MXO_P_ENV_RELEASE][v], (long)b->p[MXO_P_ENV_HOLDTIME][v], trig);
            }
            switch (c.filt_kind) {
                case MXO_FILT_LORES: x = r.filt.lores(x, cutoff_tv ? cutoff_tv[(size_t)t * V + v] : fc[v], q[v]); break;
                case MXO_FILT_HIRES: x = r.filt.hires(x, cutoff_tv ? cutoff_tv[(size_t)t * V + v] : fc[v], q[v]); break;
                case MXO_FILT_SVF:
                    if (cutoff_tv) r.svf.setCutoff(cutoff_tv[(size_t)t * V + v]);     // the patch's per-sample setter call
                    x = r.svf.play(x, c.svf_mix[0], c.svf_mix[1], c.svf_mix[2], c.svf_mix[3]); break;
                case MXO_FILT_BIQUAD:x = r.bq.play(x); break;
                default: break;
            }
            const int dsz = delay_size_tv ? (int)delay_size_tv[(size_t)t * V + v] : (int)dsize[v];
            if (c.delay_on == 1) x = b->delays[v]->dl(x, dsz, dfb[v]);
            else if (c.delay_on == 2) x = b->delays[v]->dlFromPosition(x, dsz, dfb[v], (int)b->p[MXO_P_DELAY_POSITION][v]);
            if (out) out[(size_t)t * V + v] = x;
            if (mix) { r.mixer.stereo(x, two, pan[v]); m0 += two[0]; m1 += two[1]; }
        }
        if (mix) { mix[2 * t] = m0; mix[2 * t + 1] = m1; }
    }
    if (cutoff_tv && c.filt_kind == MXO_FILT_SVF && fc)      // the modulation lasts for this call
        for (int v = first; v < first + count; ++v) b->voices[v].svf.setCutoff(fc[v]);
    return 0;
}

int32_t mxo_bank_get_ring(void* h, int32_t v, double* dst, int32_t n) {
    RefBank* b = (RefBank*)h;
    if (!b || !b->delays || v < 0 || v >= b->V || n < 0 || n > 88200 * 8) return -1;
    memcpy(dst, b->delays[v]->memory, sizeof(double) * (size_t)n);
    return 0;
}

/* the setters themselves, run on a scratch object */
double mxo_env_attack_coeff(double ms, int32_t sr) {
    maxiSettings::setup((size_t)sr, 2, 1024); maxiEnv* e = zeroed_new<maxiEnv>(); e->setAttack(ms);
    double r = e->attack; free(e); return r;
}
double mxo_env_attack_ms_coeff(double ms, int32_t sr) {
    maxiSettings::setup((size_t)sr, 2, 1024); maxiEnv* e = zeroed_new<maxiEnv>(); e->setAttackMS(ms);
    double r = e->attack; free(e); return r;
}
double mxo_env_decay_coeff(double ms, int32_t sr) {
    maxiSettings::setup((size_t)sr, 2, 1024); maxiEnv* e = zeroed_new<maxiEnv>(); e->setDecay(ms);
    double r = e->decay; free(e); return r;
}

/* ------------------------------------------------------------------ STFT */
struct RefStft { int C, n, hop, bins; std::vector<maxiFFT*> f; };

void* mxo_stft_create(int32_t channels, int32_t fft_size, int32_t hop_size) {
    if (channels <= 0 || fft_size < 4 || (fft_size & (fft_size - 1)) || hop_size <= 0 || hop_size > fft_size) return nullptr;
    RefStft* s = new RefStft();
    s->C = channels; s->n = fft_size; s->hop = hop_size; s->bins = fft_size / 2;
    for (int c = 0; c < channels; ++c) { maxiFFT* f = new maxiFFT(); f->setup(fft_size, hop_size, fft_size); s->f.push_back(f); }
    return s;
}
void mxo_stft_destroy(void* h) { RefStft* s = (RefStft*)h; if (!s) return; for (auto* f : s->f) delete f; delete s; }

int32_t mxo_stft_process(void* h, const float* in, int32_t n, int32_t max_frames,
                         float* mags, float* phases, float* re, float* im) {
    RefStft* s = (RefStft*)h;
    if (!s || !in || n < 0) return -1;
    int frames = 0;
    for (int c = 0; c < s->C; ++c) {
        maxiFFT* f = s->f[c];
        int k = 0;
        for (int t = 0; t < n; ++t) {
            if (f->process(in[(size_t)c * n + t], maxiFFT::WITH_POLAR_CONVERSION)) {
                if (k >= max_frames) return -3;
                size_t o = ((size_t)c * max_frames + k) * s->bins;
                if (mags)   memcpy(mags + o, f->getMagnitudes().data(), sizeof(float) * s->bins);
                if (phases) memcpy(phases + o, f->getPhases().data(), sizeof(float) * s->bins);
                if (re)     memcpy(re + o, f->getReal(), sizeof(float) * s->bins);
                if (im)     memcpy(im + o, f->getImag(), sizeof(float) * s->bins);
                ++k;
            }
        }
        frames = k;
    }
    return frames;
}
int32_t mxo_stft_window(void* h, float* w) {
    RefStft* s = (RefStft*)h; if (!s || !w) return -1;
    memcpy(w, s->f[0]->window.data(), sizeof(float) * s->n); return 0;
}

/* the reference methods themselves, run on a maxiFFT whose (private) magnitudes vector is loaded with each frame */
int32_t mxo_spectral_features(const float* mags, int32_t n_frames, int32_t fft_size, int32_t sample_rate,
                              float* db, float* flatness, float* centroid) {
    if (!mags || n_frames < 0 || fft_size < 4 || (fft_size & (fft_size - 1))) return -1;
    maxiSettings::setup((size_t)sample_rate, 2, 1024);
    maxiFFT f;
    f.setup(fft_size, fft_size / 2, fft_size);
    const int bins = fft_size / 2;
    for (int i = 0; i < n_frames; ++i) {
        memcpy(f.magnitudes.data(), mags + (size_t)i * bins, sizeof(float) * bins);
        f.recalc = true;
        if (db) memcpy(db + (size_t)i * bins, f.getMagnitudesDB().data(), sizeof(float) * bins);
        if (flatness) flatness[i] = f.spectralFlatness();
        if (centroid) centroid[i] = f.spectralCentroid();
    }
    return 0;
}

/* ------------------------------------------------------------------ MFCC */
struct RefMfcc { int bins, filters, coeffs; maxiMFCC m; std::vector<float> spec; };

void* mxo_mfcc_create(int32_t num_bins, int32_t num_filters, int32_t num_coeffs,
                      double min_freq, double max_freq, int32_t sample_rate) {
    if (num_bins <= 0 || num_filters <= 0 || num_coeffs <= 0) return nullptr;
    maxiSettings::setup((size_t)sample_rate, 2, 1024);
    RefMfcc* m = new RefMfcc();
    m->bins = num_bins; m->filters = num_filters; m->coeffs = num_coeffs;
    m->m.setup(num_bins, num_filters, num_coeffs, min_freq, max_freq);
    /* calcMelFilterBank never writes filter 0 (loop starts at 1, src/libs/maxiMFCC.h:149): the column is
     * whatever malloc returned. Define it as zero (what a fresh mmap'ed block holds), SURVEY.md A13. */
    for (int bin = 0; bin < num_bins; ++bin) m->m.melFilters[(size_t)bin * num_filters] = 0.0;
    m->spec.resize(num_bins);
    return m;
}
void mxo_mfcc_destroy(void* h) { delete (RefMfcc*)h; }

int32_t mxo_mfcc_process(void* h, const float* mags, int32_t n, double* coeffs, double* melbands) {
    RefMfcc* m = (RefMfcc*)h;
    if (!m || !mags || !coeffs) return -1;
    for (int i = 0; i < n; ++i) {
        memcpy(m->spec.data(), mags + (size_t)i * m->bins, sizeof(float) * m->bins);
        std::vector<double>& r = m->m.mfcc(m->spec);
        memcpy(coeffs + (size_t)i * m->coeffs, r.data(), sizeof(double) * m->coeffs);
        if (melbands) memcpy(melbands + (size_t)i * m->filters, m->m.melBands, sizeof(double) * m->filters);
    }
    return 0;
}

/* ------------------------------------------------------------------ ISTFT */
struct RefIstft { int C, n, hop, bins; std::vector<maxiIFFT*> f; std::vector<float> mg, ph; };

void* mxo_istft_create(int32_t channels, int32_t fft_size, int32_t hop_size) {
    if (channels <= 0 || fft_size < 4 || (fft_size & (fft_size - 1)) || hop_size <= 0 || hop_size > fft_size) return nullptr;
    RefIstft* s = new RefIstft();
    s->C = channels; s->n = fft_size; s->hop = hop_size; s->bins = fft_size / 2;
    for (int c = 0; c < channels; ++c) { maxiIFFT* f = new maxiIFFT(); f->setup(fft_size, hop_size, fft_size); s->f.push_back(f); }
    s->mg.resize(s->bins); s->ph.resize(s->bins);
    return s;
}
void mxo_istft_destroy(void* h) { RefIstft* s = (RefIstft*)h; if (!s) return; for (auto* f : s->f) delete f; delete s; }

int32_t mxo_istft_process(void* h, const float* mags, const float* phases, int32_t frames, float* out) {
    RefIstft* s = (RefIstft*)h;
    if (!s || !mags || !phases || !out || frames < 0) return -1;
    for (int c = 0; c < s->C; ++c) {
        for (int f = 0; f < frames; ++f) {
            size_t o = ((size_t)c * frames + f) * s->bins;
            memcpy(s->mg.data(), mags + o, sizeof(float) * s->bins);
            memcpy(s->ph.data(), phases + o, sizeof(float) * s->bins);
            for (int t = 0; t < s->hop; ++t)
                out[(size_t)c * frames * s->hop + (size_t)f * s->hop + t] = s->f[c]->process(s->mg, s->ph, maxiIFFT::SPECTRUM);
        }
    }
    return 0;
}

/* The reference's per-sample analysis / resynthesis idiom, literally (its feature-extractor examples): every sample goes into
 * maxiFFT::process(); maxiIFFT::process() is called on EVERY sample with the transform's current magnitudes / phases (it reads them on the
 * first sample of each hop). fired[i] = 1 where process() returned true. Pins what the per-sample signatures of include/maximilian_b200.hpp
 * must deliver (tests/test_oracle_vs_reference.py composes the block functions the same way). Reference library only. */
int32_t mxo_ref_per_sample_roundtrip(const float* in, int32_t n, int32_t fft_size, int32_t hop_size, float* out, uint8_t* fired) {
    if (!in || !out || !fired || n < 0) return -1;
    maxiFFT f; f.setup(fft_size, hop_size, fft_size);
    maxiIFFT g; g.setup(fft_size, hop_size, fft_size);
    int frames = 0;
    for (int i = 0; i < n; ++i) {
        const bool fr = f.process(in[i], maxiFFT::WITH_POLAR_CONVERSION);
        fired[i] = fr ? 1 : 0;
        frames += fr ? 1 : 0;
        out[i] = g.process(f.getMagnitudes(), f.getPhases(), maxiIFFT::SPECTRUM);
    }
    return frames;
}

}  // extern "C"

/* ------------------------------------------------------------------ patches
 * The same stage list as the port's interpreter (oracle_api.h), every stage being a call of the reference method on a
 * reference object that lives in zero-filled storage, one object per (stage, voice). No DSP of its own. */
namespace {

struct RefStageObj {
    maxiOsc osc; maxiEnv env; maxiFilter filt; maxiSVF svf; maxiBiquad bq; maxiDCBlocker dc; maxiNonlinearity nl; maxiMix mixer;
};

struct RefPatch {
    mxo_patch_desc d;
    std::vector<mxo_stage> stages;
    std::vector<double> consts;
    std::vector<std::vector<double>> params;
    std::vector<RefStageObj*> objs;            /* [stage] -> calloc'ed array of V objects (light stages) */
    std::vector<maxiDelayline**> delays;       /* [stage] -> V delay lines (5.6 MB each) or null */
    std::vector<maxiFlanger**> flangers;
    std::vector<maxiChorus**> choruses;        /* two delay lines each */
    std::vector<maxiEnvGen*> envgens;          /* [stage] -> array of V */
};

int ref_state_slots(const mxo_stage& g) {
    switch (g.op) {
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

/* address of state slot `slot` of stage `si`, voice v, inside the reference object (nullptr: integer / bool members, handled apart) */
double* ref_slot_ptr(RefPatch* p, int si, int slot, int v) {
    const mxo_stage& g = p->stages[si];
    RefStageObj* o = p->objs[si] ? &p->objs[si][v] : nullptr;
    switch (g.op) {
        case MXO_OP_OSC: return slot == 0 ? &o->osc.phase : &o->osc.output;
        case MXO_OP_ENV_ADSR: case MXO_OP_ENV_AR: return slot == 0 ? &o->env.amplitude : slot == 1 ? &o->env.output : nullptr;
        case MXO_OP_FILTER:
            if (g.kind == MXO_FILT_LORES || g.kind == MXO_FILT_HIRES) return slot == 0 ? &o->filt.x : &o->filt.y;
            if (g.kind == MXO_FILT_BANDPASS) return slot == 0 ? &o->filt.outputs[1] : &o->filt.outputs[2];
            return slot == 0 ? &o->filt.outputs[0] : nullptr;
        case MXO_OP_SVF: return slot == 0 ? &o->svf.v0z : slot == 1 ? &o->svf.v1 : &o->svf.v2;
        case MXO_OP_BIQUAD: return slot == 0 ? &o->bq.v[1] : &o->bq.v[2];
        case MXO_OP_DCBLOCK: return slot == 0 ? &o->dc.xm1 : &o->dc.ym1;
        case MXO_OP_FLANGER: return slot == 1 ? &p->flangers[si][v]->lfo.phase : slot == 2 ? &p->flangers[si][v]->lfo.output : nullptr;
        case MXO_OP_CHORUS: return slot == 2 ? &p->choruses[si][v]->lopass.x : slot == 3 ? &p->choruses[si][v]->lopass.y : nullptr;
        default: return nullptr;
    }
}

}  // namespace

extern "C" {

int32_t mxo_set_tables(const double*, const double*, double) { return 0; }     /* the reference has its own */
int32_t mxo_get_tables(double* sine514, double* transition1001, double* sine_before) {
    memcpy(sine514, sineBuffer, sizeof(double) * 514);
    memcpy(transition1001, transition, sizeof(double) * 1001);
    *sine_before = (&sineBuffer[0])[-1];       /* what sinebuf4 reads on its wrap sample in THIS build of the reference */
    return 0;
}

void* mxo_patch_create(const mxo_patch_desc* d) {
    if (!d || d->voices <= 0 || d->n_stages <= 0 || d->n_stages > 64 || !d->stages || !mxo_patch_shapes_ok(d)) return nullptr;
    maxiSettings::setup((size_t)d->sample_rate, 2, 1024);
    RefPatch* p = new RefPatch();
    p->d = *d;
    p->d.shapes = nullptr;                                               /* each stage's maxiEnvGen objects are set up below */
    p->stages.assign(d->stages, d->stages + d->n_stages);
    p->consts.assign(64, 0.0);
    for (int i = 0; i < d->n_consts; ++i) p->consts[i] = d->consts[i];
    p->params.assign((size_t)d->n_params, std::vector<double>((size_t)d->voices, 0.0));
    const int V = d->voices;
    for (int si = 0; si < d->n_stages; ++si) {
        const mxo_stage& g = p->stages[si];
        RefStageObj* o = (RefStageObj*)calloc((size_t)V, sizeof(RefStageObj));
        for (int v = 0; v < V; ++v) new (&o[v]) RefStageObj();
        p->objs.push_back(o);
        maxiDelayline** dl = nullptr; maxiFlanger** fl = nullptr; maxiChorus** ch = nullptr; maxiEnvGen* eg = nullptr;
        if (g.op == MXO_OP_CHORUS) { ch = (maxiChorus**)calloc((size_t)V, sizeof(void*)); for (int v = 0; v < V; ++v) ch[v] = zeroed_new<maxiChorus>(); }
        if (g.op == MXO_OP_DELAY) { dl = (maxiDelayline**)calloc((size_t)V, sizeof(void*)); for (int v = 0; v < V; ++v) dl[v] = zeroed_new<maxiDelayline>(); }
        if (g.op == MXO_OP_FLANGER) { fl = (maxiFlanger**)calloc((size_t)V, sizeof(void*)); for (int v = 0; v < V; ++v) fl[v] = zeroed_new<maxiFlanger>(); }
        if (g.op == MXO_OP_ENVGEN) {
            const mxo_envgen_shape& s = d->shapes[g.kind];
            eg = new maxiEnvGen[V];
            std::vector<double> levels(s.levels, s.levels + s.stages + 1), times(s.times, s.times + s.stages), curves(s.curves, s.curves + s.stages);
            std::streambuf* old = std::cout.rdbuf(nullptr);              /* setup() prints every segment */
            for (int v = 0; v < V; ++v) eg[v].setup(levels, times, curves, s.loop != 0, s.retrigger != 0);
            std::cout.rdbuf(old);
        }
        p->delays.push_back(dl); p->flangers.push_back(fl); p->choruses.push_back(ch); p->envgens.push_back(eg);
    }
    return p;
}

void mxo_patch_destroy(void* h) {
    RefPatch* p = (RefPatch*)h; if (!p) return;
    for (size_t si = 0; si < p->stages.size(); ++si) {
        free(p->objs[si]);
        if (p->delays[si]) { for (int v = 0; v < p->d.voices; ++v) free(p->delays[si][v]); free(p->delays[si]); }
        if (p->flangers[si]) { for (int v = 0; v < p->d.voices; ++v) free(p->flangers[si][v]); free(p->flangers[si]); }
        if (p->choruses[si]) { for (int v = 0; v < p->d.voices; ++v) free(p->choruses[si][v]); free(p->choruses[si]); }
        delete[] p->envgens[si];
    }
    delete p;
}

int32_t mxo_patch_set_param(void* h, int32_t j, const double* x) {
    RefPatch* p = (RefPatch*)h; if (!p || !x || j < 0 || j >= p->d.n_params) return -1;
    p->params[j].assign(x, x + p->d.voices);
    return 0;
}

int32_t mxo_patch_set_state(void* h, int32_t stage, int32_t slot, const double* x) {
    RefPatch* p = (RefPatch*)h;
    if (!p || !x || stage < 0 || stage >= p->d.n_stages || slot < 0 || slot >= ref_state_slots(p->stages[stage])) return -1;
    for (int v = 0; v < p->d.voices; ++v) { double* q = ref_slot_ptr(p, stage, slot, v); if (!q) return -3; *q = x[v]; }
    return 0;
}

int32_t mxo_patch_get_state(void* h, int32_t stage, int32_t slot, double* x) {
    RefPatch* p = (RefPatch*)h;
    if (!p || !x || stage < 0 || stage >= p->d.n_stages || slot < 0 || slot >= ref_state_slots(p->stages[stage])) return -1;
    const mxo_stage& g = p->stages[stage];
    for (int v = 0; v < p->d.voices; ++v) {
        double* q = ref_slot_ptr(p, stage, slot, v);
        if (q) { x[v] = *q; continue; }
        if (g.op == MXO_OP_ENV_ADSR || g.op == MXO_OP_ENV_AR) {
            maxiEnv& e = p->objs[stage][v].env;
            x[v] = slot == 2 ? (double)e.holdcount
                             : (double)((e.attackphase & 1) | (e.decayphase & 1) << 1 | (e.sustainphase & 1) << 2 | (e.holdphase & 1) << 3 | (e.releasephase & 1) << 4);
        } else if (g.op == MXO_OP_DELAY) x[v] = (double)p->delays[stage][v]->phase;
        else if (g.op == MXO_OP_FLANGER) x[v] = (double)p->flangers[stage][v]->dl.phase;
        else if (g.op == MXO_OP_CHORUS) x[v] = (double)(slot == 0 ? p->choruses[stage][v]->dl.phase : p->choruses[stage][v]->dl2.phase);
        else if (g.op == MXO_OP_ENVGEN) {
            maxiEnvGen& e = p->envgens[stage][v];
            switch (slot) {
                case 0: x[v] = e.envval; break;
                case 1: x[v] = (double)e.phase; break;
                case 2: x[v] = (double)(int)e.state; break;
                case 3: x[v] = e.nxcHappened ? 1.0 : 0.0; break;
                case 4: x[v] = e.phase < e.stages.size() ? (double)e.stages[e.phase].counter : 0.0; break;
                case 5: x[v] = e.phase < e.stages.size() ? e.stages[e.phase].currentlevel : 0.0; break;
                case 6: x[v] = e.trigDetector.previousValue; break;
                case 7: x[v] = e.trigDetector.firstTrigger ? 1.0 : 0.0; break;
                case 8: x[v] = e.holdDetector.previousValue; break;
                case 9: x[v] = e.holdDetector.firstTrigger ? 1.0 : 0.0; break;
                case 10: x[v] = e.retriggerDetector.previousValue; break;
                default: x[v] = e.retriggerDetector.firstTrigger ? 1.0 : 0.0; break;
            }
        } else return -3;
    }
    return 0;
}

int32_t mxo_patch_get_ring(void* h, int32_t stage, int32_t v, double* dst, int32_t n) {
    RefPatch* p = (RefPatch*)h;
    if (!p || !dst || stage < 0 || stage >= p->d.n_stages || v < 0 || v >= p->d.voices || n < 0 || n > 88200 * 8) return -1;
    if (p->delays[stage]) memcpy(dst, p->delays[stage][v]->memory, sizeof(double) * (size_t)n);
    else if (p->flangers[stage]) memcpy(dst, p->flangers[stage][v]->dl.memory, sizeof(double) * (size_t)n);
    else if (p->choruses[stage]) {          /* the two lines back to back, delay_taps slots of each */
        const int taps = p->d.delay_taps;
        if (n > 2 * taps) return -1;
        memcpy(dst, p->choruses[stage][v]->dl.memory, sizeof(double) * (size_t)(n < taps ? n : taps));
        if (n > taps) memcpy(dst + taps, p->choruses[stage][v]->dl2.memory, sizeof(double) * (size_t)(n - taps));
    }
    else return -1;
    return 0;
}

/* maxiOsc::noise() as the reference's own object produces it, after srand(seed) */
void mxo_srand(uint32_t seed) { srand(seed); }
void mxo_noise_fill(uint32_t seed, int64_t n, double* out) {
    srand(seed);
    maxiOsc o;
    for (int64_t i = 0; i < n; ++i) out[i] = o.noise();
}

int32_t mxo_patch_process(void* h, int32_t nframes, const double* const* inputs, double* out, double* mix) {
    RefPatch* p = (RefPatch*)h;
    if (!p || nframes < 0) return -1;
    maxiSettings::setup((size_t)p->d.sample_rate, 2, 1024);
    const size_t V = (size_t)p->d.voices;
    std::vector<double> two(2, 0.0);
    double reg[16];
    for (int t = 0; t < nframes; ++t) {
        double m0 = 0.0, m1 = 0.0;
        for (size_t v = 0; v < V; ++v) {
            for (double& r : reg) r = 0.0;
            auto F = [&](int s) -> double {
                if (s < 0) return 0.0;
                const int k = s & 0xff;
                switch (s >> 8) {
                    case 0: return reg[k];
                    case 1: return p->params[k][v];
                    case 2: return p->consts[k];
                    default: return inputs[k][(size_t)t * V + v];
                }
            };
            for (int si = 0; si < p->d.n_stages; ++si) {
                const mxo_stage& g = p->stages[si];
                RefStageObj& o = p->objs[si][v];
                double y = 0.0;
                switch (g.op) {
                    case MXO_OP_OSC:
                        switch (g.kind) {
                            case MXO_OSC_SINEBUF: y = o.osc.sinebuf(F(g.src[0])); break;
                            case MXO_OSC_SINEBUF4: y = o.osc.sinebuf4(F(g.src[0])); break;
                            case MXO_OSC_SAWN: y = o.osc.sawn(F(g.src[0])); break;
                            default: y = run_osc(o.osc, g.kind, F(g.src[0]), F(g.src[1]), F(g.src[1]), F(g.src[2])); break;
                        }
                        break;
                    case MXO_OP_ENV_ADSR:
                        y = o.env.adsr(F(g.src[0]), F(g.src[2]), F(g.src[3]), F(g.src[4]), F(g.src[5]), (long)F(g.src[6]), (int)F(g.src[1]));
                        break;
                    case MXO_OP_ENV_AR:
                        y = o.env.ar(F(g.src[0]), F(g.src[2]), F(g.src[3]), (long)F(g.src[4]), (int)F(g.src[1]));
                        break;
                    case MXO_OP_ENVGEN: y = p->envgens[si][v].play(F(g.src[0])); break;
                    case MXO_OP_FILTER:
                        switch (g.kind) {
                            case MXO_FILT_LORES: y = o.filt.lores(F(g.src[0]), F(g.src[1]), F(g.src[2])); break;
                            case MXO_FILT_HIRES: y = o.filt.hires(F(g.src[0]), F(g.src[1]), F(g.src[2])); break;
                            case MXO_FILT_LOPASS: y = o.filt.lopass(F(g.src[0]), F(g.src[1])); break;
                            case MXO_FILT_HIPASS: y = o.filt.hipass(F(g.src[0]), F(g.src[1])); break;
                            default: y = o.filt.bandpass(F(g.src[0]), F(g.src[1]), F(g.src[2])); break;
                        }
                        break;
                    case MXO_OP_SVF:
                        o.svf.setCutoff(F(g.src[1])); o.svf.setResonance(F(g.src[2]));
                        y = o.svf.play(F(g.src[0]), F(g.src[3]), F(g.src[4]), F(g.src[5]), F(g.src[6]));
                        break;
                    case MXO_OP_BIQUAD:
                        o.bq.set((maxiBiquad::filterTypes)g.kind, F(g.src[1]), F(g.src[2]), F(g.src[3]));
                        y = o.bq.play(F(g.src[0]));
                        break;
                    case MXO_OP_DCBLOCK: y = o.dc.play(F(g.src[0]), F(g.src[1])); break;
                    case MXO_OP_NONLIN:
                        switch (g.kind) {
                            case MXO_NL_ATANDIST: y = o.nl.atanDist(F(g.src[0]), F(g.src[1])); break;
                            case MXO_NL_FASTATANDIST: y = o.nl.fastAtanDist(F(g.src[0]), F(g.src[1])); break;
                            case MXO_NL_SOFTCLIP: y = o.nl.softclip(F(g.src[0])); break;
                            case MXO_NL_HARDCLIP: y = o.nl.hardclip(F(g.src[0])); break;
                            case MXO_NL_ASYMCLIP: y = o.nl.asymclip(F(g.src[0]), F(g.src[1]), F(g.src[2])); break;
                            default: y = o.nl.fastatan(F(g.src[0])); break;
                        }
                        break;
                    case MXO_OP_DELAY:
                        if (g.kind == 1) y = p->delays[si][v]->dlFromPosition(F(g.src[0]), (int)F(g.src[1]), F(g.src[2]), (int)F(g.src[3]));
                        else y = p->delays[si][v]->dl(F(g.src[0]), (int)F(g.src[1]), F(g.src[2]));
                        break;
                    case MXO_OP_FLANGER:
                        y = p->flangers[si][v]->flange(F(g.src[0]), (unsigned int)F(g.src[1]), F(g.src[2]), F(g.src[3]), F(g.src[4]));
                        break;
                    case MXO_OP_CHORUS:      /* the reference draws its own noise (rand()): src5 is what the caller predicted it to be (mxo_noise_fill / mxo_srand) */
                        y = p->choruses[si][v]->chorus(F(g.src[0]), (unsigned int)F(g.src[1]), F(g.src[2]), F(g.src[3]), F(g.src[4]));
                        break;
                    case MXO_OP_ADD: y = F(g.src[0]) + F(g.src[1]); break;
                    case MXO_OP_SUB: y = F(g.src[0]) - F(g.src[1]); break;
                    case MXO_OP_MUL: y = F(g.src[0]) * F(g.src[1]); break;
                    case MXO_OP_DIV: y = F(g.src[0]) / F(g.src[1]); break;
                    case MXO_OP_MIX_STEREO: o.mixer.stereo(F(g.src[0]), two, F(g.src[1])); m0 += two[0]; m1 += two[1]; break;
                    case MXO_OP_OUT: if (out) out[(size_t)t * V + v] = F(g.src[0]); break;
                    default: return -2;
                }
                if (g.dst >= 0) reg[g.dst] = y;
            }
        }
        if (mix) { mix[2 * t] = m0; mix[2 * t + 1] = m1; }
    }
    return 0;
}

}  // extern "C"

/* ------------------------------------------------------------------ octave analyser / bark */
struct RefOctave { int C; std::vector<maxiFFTOctaveAnalyzer*> a; };

extern "C" {

void* mxo_octave_create(int32_t channels, float sampling_rate, int32_t n_bands, int32_t n_per_octave) {
    if (channels <= 0 || n_bands <= 0) return nullptr;
    RefOctave* o = new RefOctave(); o->C = channels;
    for (int c = 0; c < channels; ++c) {
        maxiFFTOctaveAnalyzer* a = new maxiFFTOctaveAnalyzer();
        a->setup(sampling_rate, n_bands, n_per_octave);
        /* averages / peaks / peakHoldTimes come from new[] uninitialised: defined as zero */
        for (int i = 0; i < a->nAverages; ++i) { a->averages[i] = 0.f; a->peaks[i] = 0.f; a->peakHoldTimes[i] = 0; }
        o->a.push_back(a);
    }
    return o;
}
void mxo_octave_destroy(void* h) { RefOctave* o = (RefOctave*)h; if (!o) return; for (auto* a : o->a) delete a; delete o; }
int32_t mxo_octave_n_averages(void* h) { return h ? ((RefOctave*)h)->a[0]->nAverages : -1; }
int32_t mxo_octave_config(void* h, int32_t hold, float decay, float intercept, float slope) {
    RefOctave* o = (RefOctave*)h; if (!o) return -1;
    for (auto* a : o->a) { a->peakHoldTime = hold; a->peakDecayRate = decay; a->linearEQIntercept = intercept; a->linearEQSlope = slope; }
    return 0;
}
int32_t mxo_octave_process(void* h, const float* mags, int32_t frames, float* averages, float* peaks) {
    RefOctave* o = (RefOctave*)h;
    if (!o || !mags || frames < 0) return -1;
    for (int c = 0; c < o->C; ++c) {
        maxiFFTOctaveAnalyzer* a = o->a[c];
        const int nA = a->nAverages, nS = a->nSpectrum;
        std::vector<float> frame((size_t)nS);
        for (int f = 0; f < frames; ++f) {
            memcpy(frame.data(), mags + ((size_t)c * frames + f) * nS, sizeof(float) * nS);
            a->calculate(frame.data());
            if (averages) memcpy(averages + ((size_t)c * frames + f) * nA, a->averages, sizeof(float) * nA);
            if (peaks) memcpy(peaks + ((size_t)c * frames + f) * nA, a->peaks, sizeof(float) * nA);
        }
    }
    return 0;
}

#pragma GCC push_options
#pragma GCC optimize ("O0")
int32_t mxo_bark(const float* spectrum, int32_t n_frames, int32_t sample_rate, int32_t buffer_size, double* specific, double* relative, double* total) {
    if (!spectrum || n_frames < 0 || buffer_size < 4 || buffer_size / 2 > 2048) return -1;
    /* setup() writes bbLimits[24], one int past the array, into the member behind it: give the object room */
    struct Room { maxiBark b; int pad[8]; };
    Room* r = (Room*)calloc(1, sizeof(Room));
    r->b.setup((unsigned)sample_rate, (unsigned)buffer_size);
    const int spec = buffer_size / 2;
    std::vector<float> frame((size_t)spec);
    for (int f = 0; f < n_frames; ++f) {
        memcpy(frame.data(), spectrum + (size_t)f * spec, sizeof(float) * spec);
        if (specific) memcpy(specific + (size_t)f * 24, r->b.specificLoudness(frame.data()), sizeof(double) * 24);
        if (relative) memcpy(relative + (size_t)f * 24, r->b.relativeLoudness(frame.data()), sizeof(double) * 24);
        if (total) total[f] = r->b.totalLoudness(frame.data())[0];
    }
    free(r);
    return 0;
}
#pragma GCC pop_options

}  // extern "C"
