// Every recording class of include/maximilian_b200.hpp, one named case per play() body, written in the reference's vocabulary. The
// expected meaning of each case (the bank configuration or stage list the reference's signatures call for) is in tests/cpp_classes.py.
//
//   patch_classes <case> <in.bin> <out.bin> V B NB
//   patch_classes --batch <list>            one "<case> <in.bin> <out.bin> V B NB" per line; one status line per case on stdout
//
// A bank-shaped case <name> also runs as <name>_x1: the same play() with `w * 1.0` appended, an exact identity the fused bank has no
// stage for, so that the graph runs as a voice patch.
// in.bin (doubles): sineBuffer[514], transition[1001], sine_before; then per block: NP per-voice arrays [V], the gate on[V], off[V]
// (integral values), NS per-sample streams [B][V].
// out.bin (doubles): per block out[B][V] (0 where the case renders no output), bus[B][2], fused(); then the state:
//   bank:  P_PHASE, S_OSC_OUTPUT, S_FILT_0..2, S_ENV_AMPLITUDE, S_ENV_OUTPUT, S_ENV_HOLDCOUNT, S_ENV_FLAGS, S_DELAY_PHASE [V] each,
//          n, then the ring slots [V][n] (n = 0 without a delay line);
//   patch: for stages 0..63: n_slots, slots [n_slots][V], n, ring [V][n].
// Status line: "<case> ok" or "<case> maxiError <code> <block>". MXB_PATCH_MODE=fused|interpret selects the patch kernel.
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <fstream>
#include <functional>
#include <memory>
#include <sstream>
#include <string>
#include <vector>

#include "maximilian_b200.hpp"

struct Run {
    maxiVoices& v;
    int V, B, blk;
    bool x1;                                      // the _x1 copy: append `w * 1.0`
    std::vector<std::vector<double>> P;           // per-voice arrays of this block (storage outlives every play())
    std::vector<int32_t> on, off;
    std::vector<std::vector<double>> S;           // per-sample streams [B][V]
    std::vector<double>& p(int k) { return P[(size_t)k]; }
    maxiGate gate() { return maxiGate(on, off); }
    maxiStream stream(int k) { return maxiStream(S[(size_t)k]); }
    maxiSignal id(maxiSignal w) { return x1 ? w * 1.0 : w; }
};

using Body = std::function<void(Run&)>;
struct Case {
    const char* name;
    bool bank;            // bank-shaped: must run fused (and its _x1 copy must not)
    int np, ns, cap, sr;
    bool out, mix;        // what render() is handed
    std::function<Body(maxiVoices&)> make;   // builds the case's objects, returns its play()
};

template <class... T> static std::shared_ptr<std::tuple<T...>> objs(maxiVoices& v) { return std::make_shared<std::tuple<T...>>(T(v)...); }

// oscillator kind k -> stereo at a per-voice pan (P0 frequency, P1 pan, P2 duty | startphase, P3 endphase)
static Case oscCase(const char* name, int k) {
    return {name, true, 4, 0, 0, 48000, true, true, [k](maxiVoices& v) -> Body {
        auto o = std::make_shared<maxiOsc>(v); auto m = std::make_shared<maxiMix>(v);
        return [o, m, k](Run& r) {
            maxiSignal w;
            switch (k) {
                case 0: w = o->sinewave(r.p(0)); break;
                case 1: w = o->coswave(r.p(0)); break;
                case 2: w = o->phasor(r.p(0)); break;
                case 3: w = o->saw(r.p(0)); break;
                case 4: w = o->square(r.p(0)); break;
                case 5: w = o->pulse(r.p(0), r.p(2)); break;
                case 6: w = o->impulse(r.p(0)); break;
                case 7: w = o->triangle(r.p(0)); break;
                default: w = o->phasorBetween(r.p(0), r.p(2), r.p(3)); break;
            }
            m->stereo(r.id(w), r.v.bus(), r.p(1));
        };
    }};
}

// sawtooth -> maxiBiquad::set(type, P1 cutoff, P2 Q, gain) -> stereo at P3
static Case biquadCase(const char* name, maxiBiquad::filterTypes type, double gain) {
    return {name, true, 4, 0, 0, 48000, true, true, [type, gain](maxiVoices& v) -> Body {
        auto o = std::make_shared<maxiOsc>(v); auto f = std::make_shared<maxiBiquad>(v); auto m = std::make_shared<maxiMix>(v);
        return [o, f, m, type, gain](Run& r) {
            f->set(type, r.p(1), r.p(2), gain);
            maxiSignal w = f->play(o->saw(r.p(0)));
            m->stereo(r.id(w), r.v.bus(), r.p(3));
        };
    }};
}

static std::vector<Case> cases() {
    std::vector<Case> c;
    const char* oscNames[9] = {"osc_sinewave", "osc_coswave", "osc_phasor", "osc_saw", "osc_square", "osc_pulse", "osc_impulse", "osc_triangle", "osc_phasorbetween"};
    for (int k = 0; k < 9; ++k) c.push_back(oscCase(oscNames[k], k));

    // saw -> ar(P1 attack, P2 release, P3 holdtime, gate) -> lores(P4, P5) -> out only
    c.push_back({"saw_ar_lores_out", true, 6, 0, 0, 48000, true, false, [](maxiVoices& v) -> Body {
        auto o = std::make_shared<maxiOsc>(v); auto e = std::make_shared<maxiEnv>(v); auto f = std::make_shared<maxiFilter>(v);
        return [o, e, f](Run& r) {
            maxiSignal w = o->saw(r.p(0));
            w = e->ar(w, r.p(1), r.p(2), r.p(3), r.gate());
            w = f->lores(w, r.p(4), r.p(5));
            r.v.out(r.id(w));
        };
    }});
    // square -> adsr(P1 attack, P2 decay, P3 sustain, P4 release, holdtime 3, gate) -> hires(P5, P6) -> stereo at P7, bus only
    c.push_back({"square_adsr_hires_bus", true, 8, 0, 0, 48000, false, true, [](maxiVoices& v) -> Body {
        auto o = std::make_shared<maxiOsc>(v); auto e = std::make_shared<maxiEnv>(v); auto f = std::make_shared<maxiFilter>(v);
        auto m = std::make_shared<maxiMix>(v);
        return [o, e, f, m](Run& r) {
            maxiSignal w = o->square(r.p(0));
            w = e->adsr(w, r.p(1), r.p(2), r.p(3), r.p(4), 3, r.gate());
            w = f->hires(w, r.p(5), r.p(6));
            m->stereo(r.id(w), r.v.bus(), r.p(7));
        };
    }});
    c.push_back(biquadCase("biquad_lowpass", maxiBiquad::LOWPASS, 0.0));
    c.push_back(biquadCase("biquad_highpass", maxiBiquad::HIGHPASS, 0.0));
    c.push_back(biquadCase("biquad_bandpass", maxiBiquad::BANDPASS, 0.0));
    c.push_back(biquadCase("biquad_notch", maxiBiquad::NOTCH, 0.0));
    c.push_back(biquadCase("biquad_peak_p6", maxiBiquad::PEAK, 6.0));
    c.push_back(biquadCase("biquad_peak_m6", maxiBiquad::PEAK, -6.0));
    c.push_back(biquadCase("biquad_lowshelf_p6", maxiBiquad::LOWSHELF, 6.0));
    c.push_back(biquadCase("biquad_lowshelf_m6", maxiBiquad::LOWSHELF, -6.0));
    c.push_back(biquadCase("biquad_highshelf_p6", maxiBiquad::HIGHSHELF, 6.0));
    c.push_back(biquadCase("biquad_highshelf_m6", maxiBiquad::HIGHSHELF, -6.0));
    // triangle -> ADSR from setAttackMS(P1) / setDecay(P2) / setSustain(P3) / setRelease(P4) -> SVF(P5, P6) mixing (0.3, 0.2, 0.4, 0.1)
    // -> dlFromPosition(P7 size, P8 feedback, P9 position) -> stereo at P10
    c.push_back({"tri_adsr_svf_dlpos", true, 11, 0, 256, 48000, true, true, [](maxiVoices& v) -> Body {
        auto o = std::make_shared<maxiOsc>(v); auto e = std::make_shared<maxiEnv>(v); auto f = std::make_shared<maxiSVF>(v);
        auto d = std::make_shared<maxiDelayline>(v, 256); auto m = std::make_shared<maxiMix>(v);
        return [o, e, f, d, m](Run& r) {
            e->setAttackMS(r.p(1)); e->setDecay(r.p(2)); e->setSustain(r.p(3)); e->setRelease(r.p(4));
            f->setCutoff(r.p(5)); f->setResonance(r.p(6));
            maxiSignal w = o->triangle(r.p(0));
            w = e->adsr(w, r.gate());
            w = f->play(w, 0.3, 0.2, 0.4, 0.1);
            w = d->dlFromPosition(w, r.p(7), r.p(8), r.p(9));
            m->stereo(r.id(w), r.v.bus(), r.p(10));
        };
    }});
    // saw -> maxiVoices::sum
    c.push_back({"saw_sum", true, 1, 0, 0, 48000, true, true, [](maxiVoices& v) -> Body {
        auto o = std::make_shared<maxiOsc>(v);
        return [o](Run& r) { r.v.sum(r.id(o->saw(r.p(0)))); };
    }});
    // phasor with a per-voice phaseReset(P1) before blocks 0 and 2 -> stereo at P2
    c.push_back({"phasor_phase_reset", true, 3, 0, 0, 48000, true, true, [](maxiVoices& v) -> Body {
        auto o = std::make_shared<maxiOsc>(v); auto m = std::make_shared<maxiMix>(v);
        return [o, m](Run& r) {
            if (r.blk != 1) o->phaseReset(r.p(1));
            m->stereo(r.id(o->phasor(r.p(0))), r.v.bus(), r.p(2));
        };
    }});
    // saw -> a maxiSVF whose setCutoff / setResonance were never called -> stereo at P1
    c.push_back({"saw_default_svf", true, 2, 0, 0, 48000, true, true, [](maxiVoices& v) -> Body {
        auto o = std::make_shared<maxiOsc>(v); auto f = std::make_shared<maxiSVF>(v); auto m = std::make_shared<maxiMix>(v);
        return [o, f, m](Run& r) { m->stereo(r.id(f->play(o->saw(r.p(0)), 1, 0, 0, 0)), r.v.bus(), r.p(1)); };
    }});
    // at 44.1 kHz: sinewave -> ADSR from setAttack(P1) / setDecay(P2) / setSustain(0.6) / setRelease(P3) / setHoldtime(P4)
    // -> lores(P5, P6) -> dl(P7 size, P8 feedback) -> stereo at P9
    c.push_back({"sine_adsr_lores_dl_44k", true, 10, 0, 128, 44100, true, true, [](maxiVoices& v) -> Body {
        auto o = std::make_shared<maxiOsc>(v); auto e = std::make_shared<maxiEnv>(v); auto f = std::make_shared<maxiFilter>(v);
        auto d = std::make_shared<maxiDelayline>(v, 128); auto m = std::make_shared<maxiMix>(v);
        return [o, e, f, d, m](Run& r) {
            e->setAttack(r.p(1)); e->setDecay(r.p(2)); e->setSustain(0.6); e->setRelease(r.p(3)); e->setHoldtime(r.p(4));
            maxiSignal w = e->adsr(o->sinewave(r.p(0)), r.gate());
            w = f->lores(w, r.p(5), r.p(6));
            w = d->dl(w, r.p(7), r.p(8));
            m->stereo(r.id(w), r.v.bus(), r.p(9));
        };
    }});
    // per-voice frequency P0, cutoff P1 and pan P3 that change on block 1 and stay on block 2: saw -> lores -> stereo
    c.push_back({"block_params", true, 4, 0, 0, 48000, true, true, [](maxiVoices& v) -> Body {
        auto o = std::make_shared<maxiOsc>(v); auto f = std::make_shared<maxiFilter>(v); auto m = std::make_shared<maxiMix>(v);
        return [o, f, m](Run& r) { m->stereo(r.id(f->lores(o->saw(r.p(0)), r.p(1), r.p(2))), r.v.bus(), r.p(3)); };
    }});
    // gates that start before the block, end after it, are empty (on >= off), or absent: saw -> adsr(P1..P4 raw, holdtime 2) -> out
    c.push_back({"gate_edges", true, 5, 0, 0, 48000, true, false, [](maxiVoices& v) -> Body {
        auto o = std::make_shared<maxiOsc>(v); auto e = std::make_shared<maxiEnv>(v);
        return [o, e](Run& r) { r.v.out(r.id(e->adsr(o->saw(r.p(0)), r.p(1), r.p(2), r.p(3), r.p(4), 2, r.gate()))); };
    }});
    // a constant that changes on block 1: a different patch (maxiError MXB_ERR_UNSUPPORTED)
    c.push_back({"const_change", false, 0, 0, 0, 48000, true, false, [](maxiVoices& v) -> Body {
        auto o = std::make_shared<maxiOsc>(v);
        return [o](Run& r) { r.v.out(o->saw(r.blk == 0 ? 440.0 : 330.0)); };
    }});
    // a maxiBiquad whose set() was never called (maxiError MXB_ERR_UNSUPPORTED)
    c.push_back({"biquad_unset", false, 1, 0, 0, 48000, true, false, [](maxiVoices& v) -> Body {
        auto o = std::make_shared<maxiOsc>(v); auto f = std::make_shared<maxiBiquad>(v);
        return [o, f](Run& r) { r.v.out(f->play(o->saw(r.p(0)))); };
    }});

    // ---- patch-shaped: must not run fused ----
    c.push_back({"table_oscs", false, 3, 0, 0, 48000, true, false, [](maxiVoices& v) -> Body {
        auto o = objs<maxiOsc, maxiOsc, maxiOsc>(v);
        return [o](Run& r) {
            maxiSignal a = std::get<0>(*o).sinebuf(r.p(0));
            maxiSignal b = std::get<1>(*o).sinebuf4(r.p(1));
            maxiSignal c = std::get<2>(*o).sawn(r.p(2));
            maxiSignal s = a + b;
            r.v.out(s + c);
        };
    }});
    c.push_back({"maxifilter_patch", false, 8, 0, 0, 48000, true, false, [](maxiVoices& v) -> Body {
        auto o = std::make_shared<maxiOsc>(v); auto f = objs<maxiFilter, maxiFilter, maxiFilter, maxiFilter>(v);
        return [o, f](Run& r) {
            maxiSignal x = o->saw(r.p(0));
            maxiSignal a = std::get<0>(*f).lopass(x, r.p(1));
            maxiSignal b = std::get<1>(*f).hipass(x, r.p(2));
            maxiSignal c = std::get<2>(*f).bandpass(x, r.p(3), r.p(4));
            maxiSignal d = std::get<3>(*f).hires(x, r.p(5), r.p(6));
            maxiSignal s = a + b;
            s = s + c;
            s = s + d;
            r.v.out(s * r.p(7));
        };
    }});
    c.push_back({"nonlinearities", false, 5, 0, 0, 48000, true, false, [](maxiVoices& v) -> Body {
        auto o = std::make_shared<maxiOsc>(v); auto n = std::make_shared<maxiNonlinearity>(v);
        return [o, n](Run& r) {
            maxiSignal x = o->saw(r.p(0));
            x = x * 1.5;
            maxiSignal a = n->atanDist(x, r.p(1));
            maxiSignal b = n->fastAtanDist(x, r.p(2));
            maxiSignal c = n->softclip(x);
            maxiSignal d = n->hardclip(x);
            maxiSignal e = n->asymclip(x, r.p(3), r.p(4));
            maxiSignal f = n->fastatan(x);
            maxiSignal s = a + b;
            s = s + c; s = s + d; s = s + e; s = s + f;
            r.v.out(s);
        };
    }});
    c.push_back({"dcblock_flanger_chorus", false, 9, 1, 512, 48000, true, false, [](maxiVoices& v) -> Body {
        auto o = std::make_shared<maxiOsc>(v); auto dc = std::make_shared<maxiDCBlocker>(v);
        auto fl = std::make_shared<maxiFlanger>(v, 512); auto ch = std::make_shared<maxiChorus>(v, 512);
        return [o, dc, fl, ch](Run& r) {
            maxiSignal x = o->saw(r.p(0));
            maxiSignal y = x + 0.25;
            maxiSignal a = dc->play(y, r.p(1));
            maxiSignal b = fl->flange(x, r.p(2), r.p(3), r.p(4), r.p(5));
            maxiSignal c = ch->chorus(x, 120, r.p(6), r.p(7), r.p(8), r.stream(0));
            maxiSignal s = a + b;
            r.v.out(s + c);
        };
    }});
    c.push_back({"env_triggers", false, 11, 2, 0, 48000, true, false, [](maxiVoices& v) -> Body {
        auto o = objs<maxiOsc, maxiOsc>(v); auto e = objs<maxiEnv, maxiEnv, maxiEnv>(v);
        return [o, e](Run& r) {
            maxiSignal x = std::get<0>(*o).triangle(r.p(0));
            maxiSignal a = std::get<0>(*e).adsr(x, r.p(1), r.p(2), r.p(3), r.p(4), r.p(5), r.stream(0));
            maxiSignal b = std::get<1>(*e).ar(x, r.p(6), r.p(7), r.p(8), r.stream(1));
            maxiSignal t = std::get<1>(*o).square(r.p(9));
            maxiEnv& e3 = std::get<2>(*e);
            e3.setAttackMS(2.0); e3.setDecay(20.0); e3.setSustain(0.5); e3.setRelease(30.0); e3.setHoldtime(r.p(10));
            maxiSignal c = e3.adsr(x, t);
            maxiSignal s = a + b;
            r.v.out(s + c);
        };
    }});
    c.push_back({"modulated_filters", false, 3, 0, 0, 48000, true, false, [](maxiVoices& v) -> Body {
        auto o = objs<maxiOsc, maxiOsc>(v); auto f = std::make_shared<maxiSVF>(v); auto q = std::make_shared<maxiBiquad>(v);
        return [o, f, q](Run& r) {
            maxiSignal x = std::get<0>(*o).saw(r.p(0));
            maxiSignal lfo = std::get<1>(*o).sinewave(3.0);
            maxiSignal cut = lfo * 600.0;
            cut = cut + 1500.0;
            f->setCutoff(cut); f->setResonance(r.p(1));
            maxiSignal a = f->play(x, 0.5, 0.25, 0.125, 0.0625);
            q->set(maxiBiquad::BANDPASS, 2000.0, r.p(2), 0.0);
            maxiSignal b = q->play(x);
            r.v.out(a + b);
        };
    }});
    c.push_back({"envgen_triggers", false, 2, 0, 0, 48000, true, false, [](maxiVoices& v) -> Body {
        auto o = std::make_shared<maxiOsc>(v); auto g = objs<maxiEnvGen, maxiEnvGen, maxiEnvGen, maxiEnvGen>(v);
        std::get<0>(*g).setup({0.0, 1.0, 0.3, 0.0}, {1.5, 2.0, 1.0}, {2.0, 1.0, 0.5}, false);
        std::get<0>(*g).setRetrigger(true);
        std::get<1>(*g).setupADSR(1.0, 1.0, 0.5, 2.0);
        std::get<2>(*g).setupAR(2.0, 3.0);
        std::get<2>(*g).setLoop(true);
        std::get<3>(*g).setupASR(0.5, 1.0);
        return [o, g](Run& r) {
            maxiSignal a = std::get<0>(*g).play(maxiParam(r.p(0)));
            maxiSignal t = o->square(r.p(1));
            maxiSignal b = std::get<1>(*g).play(t);
            maxiSignal c = std::get<2>(*g).play(maxiParam(r.p(0)));
            maxiSignal d = std::get<3>(*g).play(t);
            maxiSignal s = a + b;
            s = s + c;
            r.v.out(s + d);
        };
    }});
    c.push_back({"operand_order", false, 2, 0, 0, 48000, true, false, [](maxiVoices& v) -> Body {
        auto o = std::make_shared<maxiOsc>(v);
        return [o](Run& r) {
            maxiSignal w = o->saw(r.p(0));
            const std::vector<double>& p = r.p(1);
            maxiSignal a = 1.0 - w;
            maxiSignal b = w - p;
            maxiSignal c = p / w;
            maxiSignal d = w / p;
            maxiSignal e = w * w;
            maxiSignal s = a * 3.0;
            s = s + b;
            s = s * 5.0;
            s = s + c;
            s = s * 7.0;
            s = s + d;
            s = s * 11.0;
            r.v.out(s + e);
        };
    }});
    c.push_back({"stereo_and_sum", false, 3, 0, 0, 48000, true, true, [](maxiVoices& v) -> Body {
        auto o = objs<maxiOsc, maxiOsc>(v); auto m = std::make_shared<maxiMix>(v);
        return [o, m](Run& r) {
            maxiSignal a = std::get<0>(*o).saw(r.p(0));
            maxiSignal b = std::get<1>(*o).triangle(r.p(1));
            m->stereo(a, r.v.bus(), r.p(2));
            r.v.sum(b);
        };
    }});
    // two oscillators, each with its own phaseReset: osc 1 before blocks 0 and 2 (P2), osc 2 before block 1 (P3)
    c.push_back({"two_phase_resets", false, 4, 0, 0, 48000, true, false, [](maxiVoices& v) -> Body {
        auto o = objs<maxiOsc, maxiOsc>(v);
        return [o](Run& r) {
            if (r.blk != 1) std::get<0>(*o).phaseReset(r.p(2));
            if (r.blk == 1) std::get<1>(*o).phaseReset(r.p(3));
            maxiSignal a = std::get<0>(*o).phasor(r.p(0));
            maxiSignal b = std::get<1>(*o).saw(r.p(1));
            r.v.out(a + b);
        };
    }});
    return c;
}

static const int32_t kBankState[] = {MXB_P_PHASE, MXB_S_OSC_OUTPUT, MXB_S_FILT_0, MXB_S_FILT_1, MXB_S_FILT_2, MXB_S_ENV_AMPLITUDE,
                                     MXB_S_ENV_OUTPUT, MXB_S_ENV_HOLDCOUNT, MXB_S_ENV_FLAGS, MXB_S_DELAY_PHASE};

static void put(FILE* f, const double* x, size_t n) { fwrite(x, sizeof(double), n, f); }
static void put1(FILE* f, double x) { put(f, &x, 1); }

static void writeState(FILE* g, maxiVoices& v, int cap) {
    const int V = v.size();
    std::vector<double> x((size_t)V);
    if (v.fused()) {
        for (int32_t id : kBankState) {     // a state the chain does not have (no envelope, no SVF, ...): NaN
            if (mxb_bank_get_state(v.handle(), id, x.data(), MXB_MEM_HOST) != MXB_OK) std::fill(x.begin(), x.end(), std::nan(""));
            put(g, x.data(), x.size());
        }
        const int n = v.handle() && cap > 0 && mxb_bank_get_ring(v.handle(), 0, x.data(), 0, MXB_MEM_HOST) == MXB_OK ? cap : 0;
        put1(g, n);
        std::vector<double> ring((size_t)n);
        for (int k = 0; k < V && n; ++k) {
            maxib200_detail::check(mxb_bank_get_ring(v.handle(), k, ring.data(), n, MXB_MEM_HOST), "mxb_bank_get_ring");
            put(g, ring.data(), ring.size());
        }
        return;
    }
    mxb_patch* p = v.patchHandle();
    for (int st = 0; st < 64; ++st) {       // stages past the end and stages without state both have no slots
        std::vector<std::vector<double>> slots;
        while (mxb_patch_get_state(p, st, (int32_t)slots.size(), x.data(), MXB_MEM_HOST) == MXB_OK) slots.push_back(x);
        put1(g, (double)slots.size());
        for (auto& s : slots) put(g, s.data(), s.size());
        std::vector<double> ring((size_t)2 * (size_t)cap);
        int n = 0;                          // a chorus stage owns two lines, a delay or flanger stage one, any other stage none
        if (cap > 0 && mxb_patch_get_ring(p, st, 0, ring.data(), 0, MXB_MEM_HOST) == MXB_OK)
            n = mxb_patch_get_ring(p, st, 0, ring.data(), 2 * cap, MXB_MEM_HOST) == MXB_OK ? 2 * cap : cap;
        put1(g, n);
        ring.resize((size_t)n);
        for (int k = 0; k < V && n; ++k) {
            maxib200_detail::check(mxb_patch_get_ring(p, st, k, ring.data(), n, MXB_MEM_HOST), "mxb_patch_get_ring");
            put(g, ring.data(), ring.size());
        }
    }
}

static std::string runCase(const std::vector<Case>& all, std::string name, const char* inPath, const char* outPath, int V, int B, int NB) {
    bool x1 = false;
    const Case* cs = nullptr;
    for (const Case& c : all) if (name == c.name) cs = &c;
    if (!cs && name.size() > 3 && name.compare(name.size() - 3, 3, "_x1") == 0) {
        for (const Case& c : all) if (c.bank && name.compare(0, name.size() - 3, c.name) == 0) cs = &c;
        x1 = true;
    }
    if (!cs) return name + " unknown-case";
    std::ifstream in(inPath, std::ios::binary | std::ios::ate);
    if (!in) return name + " cannot-read";
    const size_t bytes = (size_t)in.tellg();
    const size_t perBlock = (size_t)cs->np * V + 2 * (size_t)V + (size_t)cs->ns * B * V;
    if (bytes != sizeof(double) * (1516 + perBlock * (size_t)NB)) return name + " bad-input-size";
    std::vector<double> data(bytes / sizeof(double));
    in.seekg(0);
    in.read(reinterpret_cast<char*>(data.data()), (std::streamsize)bytes);

    maxiSettings::setup((size_t)cs->sr, 2, (size_t)B);
    maxiVoices voices(V);
    voices.setTables(data.data(), data.data() + 514, data[1515]);
    Run r{voices, V, B, 0, x1, std::vector<std::vector<double>>((size_t)cs->np, std::vector<double>((size_t)V)), std::vector<int32_t>((size_t)V),
          std::vector<int32_t>((size_t)V), std::vector<std::vector<double>>((size_t)cs->ns, std::vector<double>((size_t)B * V))};
    FILE* g = fopen(outPath, "wb");
    if (!g) return name + " cannot-write";
    std::string status = name + " ok";
    int blk = 0;
    try {
        Body play = cs->make(voices);
        std::vector<double> out((size_t)B * V), mix((size_t)B * 2);
        for (blk = 0; blk < NB; ++blk) {
            const double* d = data.data() + 1516 + perBlock * (size_t)blk;
            for (int k = 0; k < cs->np; ++k, d += V) std::copy(d, d + V, r.P[(size_t)k].begin());
            for (int k = 0; k < V; ++k) r.on[(size_t)k] = (int32_t)d[k];
            for (int k = 0; k < V; ++k) r.off[(size_t)k] = (int32_t)d[V + k];
            d += 2 * V;
            for (int k = 0; k < cs->ns; ++k, d += (size_t)B * V) std::copy(d, d + (size_t)B * V, r.S[(size_t)k].begin());
            r.blk = blk;
            std::fill(out.begin(), out.end(), 0.0); std::fill(mix.begin(), mix.end(), 0.0);
            play(r);
            voices.render(B, cs->out ? out.data() : nullptr, cs->mix ? mix.data() : nullptr);
            put(g, out.data(), out.size()); put(g, mix.data(), mix.size()); put1(g, voices.fused() ? 1.0 : 0.0);
        }
        writeState(g, voices, cs->cap);
    } catch (const maxiError& err) {
        status = name + " maxiError " + std::to_string(err.code) + " " + std::to_string(blk);
        fprintf(stderr, "%s: %s\n", name.c_str(), err.what());
    }
    fclose(g);
    return status;
}

int main(int argc, char** argv) {
    const std::vector<Case> all = cases();
    if (argc == 2 && std::string(argv[1]) == "--list") {
        for (const Case& c : all) printf("%s %d\n", c.name, c.bank ? 1 : 0);
        return 0;
    }
    if (argc == 3 && std::string(argv[1]) == "--batch") {
        std::ifstream list(argv[2]);
        std::string line;
        while (std::getline(list, line)) {
            std::istringstream ls(line);
            std::string name, in, out; int V = 0, B = 0, NB = 0;
            if (!(ls >> name >> in >> out >> V >> B >> NB)) continue;
            printf("%s\n", runCase(all, name, in.c_str(), out.c_str(), V, B, NB).c_str());
            fflush(stdout);
        }
        return 0;
    }
    if (argc != 7) {
        fprintf(stderr, "usage: patch_classes <case> <in.bin> <out.bin> V B NB | --batch <list> | --list\n");
        return 2;
    }
    const std::string s = runCase(all, argv[1], argv[2], argv[3], atoi(argv[4]), atoi(argv[5]), atoi(argv[6]));
    printf("%s\n", s.c_str());
    return s.size() > 3 && s.compare(s.size() - 3, 3, " ok") == 0 ? 0 : 1;
}
