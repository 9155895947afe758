// The play() of cpp/commandline/maximilian_examples/16.Replicant/main.cpp over V voices, written against include/maximilian_b200.hpp: a
// metronome (maxiOsc::phasor) whose ticks fire the bass envelope for one sample, step an arpeggio (currentPitch), and on some ticks fire the
// lead envelope and step the lead line (trigger2, leadPitch). Every voice runs its own metronome, at its own tempo. The per-sample CONTROL
// half of the original play() runs on the host once per block over all of its samples, for every voice, and writes the four control values
// exactly as the original writes its globals (the pitches are floats there, and here). The audio half is recorded once per block and runs
// on the GPU. The note tables are this program's own; the lead line's output is dropped by the original (only the bass reaches output[]), so
// here it goes to the bus, to have leadPitch and trigger2 checked as well; the original's delay line feeds nothing and is left out.
//
// The same program runs twice: once with the control values handed over as maxiEvents (an event where a value changes), once as dense
// maxiStreams (every value of every sample). The two must give the same bits.
//
//   patch_events <tables.bin> <out.bin> V NBLOCKS B      tables.bin: sineBuffer[514] ++ transition[1001] ++ sine_before (doubles)
// out.bin, doubles: the four dense control streams (currentPitch, leadPitch, trigger, trigger2) [NBLOCKS * B][V] each, then for the events run
// and the dense run: output[0] (bassout / 2) [NBLOCKS * B][V] and the bus [NBLOCKS * B][2].
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <vector>

#include "maximilian_b200.hpp"

struct Replicant {
    maxiVoices v;
    maxiOsc sound, bass, mod, lead, lead2, leadmod;
    maxiEnv envelope, leadenvelope;
    maxiFilter filter, filter2;
    maxiMix mix;
    maxiEvents currentPitchEv, leadPitchEv, triggerEv, trigger2Ev;
    explicit Replicant(int V)
        : v(V), sound(v), bass(v), mod(v), lead(v), lead2(v), leadmod(v), envelope(v), leadenvelope(v), filter(v), filter2(v), mix(v),
          currentPitchEv(v), leadPitchEv(v), triggerEv(v), trigger2Ev(v) {}

    // the audio half of the original play(), one statement per call so that the recorded order does not depend on the compiler
    template <class X> void play(const X& currentPitch, const X& leadPitch, const X& trigger, const X& trigger2) {
        maxiSignal cp = v.signal(currentPitch), lp = v.signal(leadPitch);
        maxiSignal half = cp * 0.5;
        maxiSignal b = bass.saw(half);
        maxiSignal m = mod.phasor(1);
        maxiSignal s = sound.pulse(half, m);
        maxiSignal bassout = filter2.lores(envelope.adsr(b + s, 1, 0.9995, 0.25, 0.9995, 1, trigger), 9250, 2);
        maxiSignal l2 = lead2.saw(lp * 4);
        maxiSignal lm = leadmod.sinebuf(1.9);
        maxiSignal l1 = lead.pulse(lp + lm * 1.5, 0.6);
        maxiSignal leadout = filter.lores(leadenvelope.ar(l2 + l1, 0.00005, 0.999975, 50000, trigger2), 5900, 10);
        v.out(bassout);
        mix.stereo(leadout, v.bus(), 0.5);
    }
};

// one voice's control state: the original's globals
struct Control {
    double timerPhase = 0, tempo = 9;
    int lastCount = 0, playHead = 0, currentChord = 0, newnote = 0, trigger = 0, trigger2 = 0;
    float currentPitch = 0, leadPitch = 0;
};
const int kPitch[4] = {45, 48, 50, 52}, kChord[8] = {0, 5, 5, 7, 0, 3, 7, 2}, kLead[15] = {64, 62, 60, 67, 65, 64, 62, 60, 59, 57, 59, 60, 62, 64, 55};
double mtof(int m) { return 440.0 * std::pow(2.0, (m - 69) / 12.0); }
bool leadTick(int playHead) { const int k = playHead % 32; return k == 0 || k == 6 || k == 11 || k == 16 || k == 22 || k == 24; }

int main(int argc, char** argv) {
    if (argc != 6) { fprintf(stderr, "usage: patch_events tables.bin out.bin V NBLOCKS B\n"); return 2; }
    const int V = atoi(argv[3]), NB = atoi(argv[4]), B = atoi(argv[5]);
    std::vector<double> tab(514 + 1001 + 1);
    FILE* f = fopen(argv[1], "rb");
    if (!f || fread(tab.data(), sizeof(double), tab.size(), f) != tab.size()) { fprintf(stderr, "cannot read %s\n", argv[1]); return 2; }
    fclose(f);
    try {
        maxiSettings::setup(44100, 2, B);
        Replicant ev(V), de(V);
        for (Replicant* r : {&ev, &de}) r->v.setTables(tab.data(), tab.data() + 514, tab[514 + 1001]);
        std::vector<Control> ctl((size_t)V);
        for (int i = 0; i < V; ++i) ctl[(size_t)i].tempo = 9.0 + 2.5 * i;                   // every voice at its own tempo
        const size_t N = (size_t)NB * B * V;
        std::vector<double> streams[4], outE, outD, busE, busD;
        for (auto& s : streams) s.reserve(N);
        std::vector<double> dense[4], o((size_t)B * V), bus((size_t)B * 2);
        std::vector<double> lastSent((size_t)V * 4, 0.0);                                   // what the events streams hold (they start at 0.0)
        maxiEvents* evs[4] = {&ev.currentPitchEv, &ev.leadPitchEv, &ev.triggerEv, &ev.trigger2Ev};
        for (int blk = 0; blk < NB; ++blk) {
            for (auto& d : dense) d.assign((size_t)B * V, 0.0);
            for (int t = 0; t < B; ++t)
                for (int i = 0; i < V; ++i) {
                    Control& c = ctl[(size_t)i];
                    const double out = c.timerPhase;                                          // maxiOsc::phasor(tempo)
                    if (c.timerPhase >= 1.0) c.timerPhase -= 1.0;
                    c.timerPhase += (1. / (maxiSettings::sampleRate / (c.tempo)));
                    const int currentCount = (int)out;
                    if (c.lastCount != currentCount) {
                        c.trigger = 1;
                        c.trigger2 = leadTick(c.playHead) ? 1 : 0;
                        if (c.trigger2 == 1) {
                            c.leadPitch = mtof(kLead[c.newnote]);
                            c.newnote++;
                            if (c.newnote > 14) c.newnote = 0;
                        }
                        c.currentPitch = mtof(kPitch[c.playHead % 4] + kChord[c.currentChord % 8]);
                        c.playHead++;
                        if (c.playHead % 32 == 0) c.currentChord++;
                        c.lastCount = 0;
                    }
                    const double val[4] = {c.currentPitch, c.leadPitch, (double)c.trigger, (double)c.trigger2};    // what this sample reads
                    for (int k = 0; k < 4; ++k) {
                        dense[k][(size_t)t * V + i] = val[k];
                        if (val[k] != lastSent[(size_t)i * 4 + k]) { evs[k]->set(t, i, val[k]); lastSent[(size_t)i * 4 + k] = val[k]; }
                    }
                    if (c.trigger != 0) c.trigger = 0;
                }
            for (int k = 0; k < 4; ++k) streams[k].insert(streams[k].end(), dense[k].begin(), dense[k].end());
            ev.play(ev.currentPitchEv, ev.leadPitchEv, ev.triggerEv, ev.trigger2Ev);
            ev.v.render(B, o.data(), bus.data());
            for (double x : o) outE.push_back(x / 2);
            busE.insert(busE.end(), bus.begin(), bus.end());
            de.play(maxiStream(dense[0]), maxiStream(dense[1]), maxiStream(dense[2]), maxiStream(dense[3]));
            de.v.render(B, o.data(), bus.data());
            for (double x : o) outD.push_back(x / 2);
            busD.insert(busD.end(), bus.begin(), bus.end());
        }
        FILE* g = fopen(argv[2], "wb");
        if (!g) { fprintf(stderr, "cannot write %s\n", argv[2]); return 2; }
        for (auto* a : {&streams[0], &streams[1], &streams[2], &streams[3], &outE, &busE, &outD, &busD}) fwrite(a->data(), sizeof(double), a->size(), g);
        fclose(g);
    } catch (const maxiError& e) {
        fprintf(stderr, "maxiError %d: %s\n", e.code, e.what());
        return 1;
    }
    return 0;
}
