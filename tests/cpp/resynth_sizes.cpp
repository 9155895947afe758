// The reference's analysis -> resynthesis idiom, one sample per call (its 20.FFT_example and feature-extractor examples):
// `if (fft.process(x)) { ... }` and `out = ifft.process(fft.getMagnitudes(), fft.getPhases())` on every sample, against
// include/maximilian_b200.hpp, at the frame size and hop given on the command line (2048 points, hops that do not divide the frame).
//
//   resynth_sizes <in.bin> <out.bin> N fftSize hopSize
// in.bin:  N float32 samples of one channel.
// out.bin: int32 F (frames fired), float32 fired[N] (1 where fft.process returned true), float32 out[N].
#include <cstdio>
#include <cstdlib>
#include <vector>

#include "maximilian_b200.hpp"

int main(int argc, char** argv) {
    if (argc != 6) { fprintf(stderr, "usage: resynth_sizes in.bin out.bin N fftSize hopSize\n"); return 2; }
    const int N = atoi(argv[3]), fftSize = atoi(argv[4]), hopSize = atoi(argv[5]);
    vector<float> x((size_t)N);
    FILE* fi = fopen(argv[1], "rb");
    if (!fi || fread(x.data(), sizeof(float), x.size(), fi) != x.size()) { fprintf(stderr, "cannot read %s\n", argv[1]); return 1; }
    fclose(fi);
    try {
        maxiSettings::setup(44100, 1, 512);
        maxiFFT fft;
        maxiIFFT ifft;
        fft.setup(fftSize, hopSize, fftSize);
        ifft.setup(fftSize, hopSize, fftSize);
        vector<float> fired((size_t)N, 0.f), out((size_t)N);
        int32_t F = 0;
        for (int i = 0; i < N; ++i) {
            if (fft.process(x[(size_t)i])) { fired[(size_t)i] = 1.f; ++F; }
            out[(size_t)i] = ifft.process(fft.getMagnitudes(), fft.getPhases());
        }
        FILE* fo = fopen(argv[2], "wb");
        fwrite(&F, sizeof(F), 1, fo);
        fwrite(fired.data(), sizeof(float), fired.size(), fo);
        fwrite(out.data(), sizeof(float), out.size(), fo);
        fclose(fo);
    } catch (const std::exception& e) { fprintf(stderr, "%s\n", e.what()); return 1; }
    return 0;
}
