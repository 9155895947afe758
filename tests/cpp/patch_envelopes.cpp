// cpp/commandline/maximilian_examples/9.Envelopes2/main.cpp, written against include/maximilian_b200.hpp: the same objects, the same
// setup() calls and the same play() expressions. The example's two maxiPolyBLEP oscillators (third-party code, not part of this library)
// become maxiOsc::square / maxiOsc::triangle. Three maxiEnvGen objects with three different shapes: one gates the oscillators, one slowly
// widens the pulse that triggers it, one sweeps the biquad's cutoff on every sample.
//
//   patch_envelopes <out.bin> NBLOCKS B
// out.bin: output[0] of both voices, [NBLOCKS][B][2] doubles. MXB_PATCH_MODE=interpret runs the interpreting kernel.
#include <cstdio>
#include <cstdlib>
#include <vector>

#include "maximilian_b200.hpp"

// two voices of the example's mono patch
maxiVoices voices(2);
maxiOsc osc1(voices), osc2(voices), trig(voices);
maxiEnvGen myEnv(voices), myEnv2(voices), myEnv3(voices);
maxiBiquad filter(voices);

void setup() {
    myEnv.setup({0, 1, 1, 0.1}, {200, maxiEnvGen::HOLD, 200}, {1, 1, 1}, false);
    myEnv2.setup({0, 1}, {10000}, {1}, false);
    myEnv3.setup({2000, 100}, {10000}, {0.5}, false);
}

void play(maxiVoices& v) {
    maxiSignal env = myEnv.play(trig.pulse(1, myEnv2.play(1)));
    filter.set(maxiBiquad::LOWPASS, myEnv3.play(1), 2, 3);
    maxiSignal frequency = 20 + (env * 500);
    maxiSignal output0 = filter.play(osc1.square(frequency) + osc2.triangle((frequency + 25) * 2));
    v.out(output0);
}

int main(int argc, char** argv) {
    if (argc != 4) { fprintf(stderr, "usage: patch_envelopes out.bin NBLOCKS B\n"); return 2; }
    const int NB = atoi(argv[2]), B = atoi(argv[3]);
    try {
        maxiSettings::setup(44100, 2, B);
        setup();
        vector<double> output, block((size_t)B * (size_t)voices.size());
        for (int blk = 0; blk < NB; ++blk) {
            play(voices);                                         // what the audio callback does once per block
            voices.render(B, block.data(), nullptr);
            output.insert(output.end(), block.begin(), block.end());
        }
        if (voices.fused()) { fprintf(stderr, "expected a voice patch, got the fused bank\n"); return 1; }
        FILE* g = fopen(argv[1], "wb");
        fwrite(output.data(), sizeof(double), output.size(), g);
        fclose(g);
    } catch (const maxiError& err) {
        fprintf(stderr, "maxiError %d: %s\n", err.code, err.what());
        return 1;
    }
    return 0;
}
