// Attached analysers on a block transform of several channels: maxiFFT(C).process(values, nSamples) fires several frames per channel
// and call, and at sizes other than 1024 runs the octave analyser and maxiBark on the magnitudes it wrote -- every channel and frame
// at its own rows. Then the refusal of an attached octave analyser whose band count is not the transform's bin count.
//
//   featurex_block <in.bin> <out.bin> C N fftSize
// in.bin:  C x N float32 samples, planar.
// out.bin: int32 F (frames per channel), int32 nAverages, int32 refusal codes for nBandsInTheFFT = fftSize and = fftSize / 4,
//          int32 frames fired by a call after the refusals, then per channel c, frame f (in that order): float32 mags[C][F][fftSize/2],
//          averages[C][F][nAverages], peaks[C][F][nAverages], float64 specific[C][F][24], relative[C][F][24], total[C][F].
#include <cstdio>
#include <cstdlib>
#include <vector>

#include "maximilian_b200.hpp"

template <class T> static void put(FILE* f, const std::vector<T>& v) { fwrite(v.data(), sizeof(T), v.size(), f); }

static int32_t refusal(int C, int fftSize, int nBands, const std::vector<float>& x, int N) {
    maxiFFT fft(C);
    maxiFFTOctaveAnalyzer oct;
    fft.setup(fftSize, fftSize / 2, fftSize);
    oct.setup(48000, nBands, 3);
    fft.attach(oct);
    try { fft.process(x.data(), N); } catch (const maxiError& e) { return e.code; }
    return 0;
}

int main(int argc, char** argv) {
    if (argc != 6) { fprintf(stderr, "usage: featurex_block in.bin out.bin C N fftSize\n"); return 2; }
    const int C = atoi(argv[3]), N = atoi(argv[4]), fftSize = atoi(argv[5]), hop = fftSize / 2, bins = fftSize / 2;
    std::vector<float> x((size_t)C * N);
    FILE* fi = fopen(argv[1], "rb");
    if (!fi || fread(x.data(), sizeof(float), x.size(), fi) != x.size()) { fprintf(stderr, "cannot read %s\n", argv[1]); return 1; }
    fclose(fi);
    try {
        maxiSettings::setup(48000, 2, 512);
        maxiFFT fft(C);
        maxiFFTOctaveAnalyzer oct;
        maxiBark bark;
        fft.setup(fftSize, hop, fftSize);
        fft.attach(oct); fft.attach(bark);
        oct.setup(48000, bins, 6);
        bark.setup(48000, fftSize);
        oct.peakHoldTime = 3; oct.peakDecayRate = 0.85f; oct.linearEQIntercept = 1.1f; oct.linearEQSlope = 0.002f;
        std::vector<std::vector<float>> mags(C), avs(C), pks(C);
        std::vector<std::vector<double>> spec(C), rel(C), tot(C);
        // ragged calls: several frames each, maxFrames left at its default (more rows than frames fire)
        const int cuts[] = {0, 5 * hop + 37, 6 * hop + 37, 9 * hop + 11, N};
        std::vector<float> blk;
        int F = 0;
        for (int k = 0; k + 1 < (int)(sizeof(cuts) / sizeof(cuts[0])); ++k) {
            const int lo = cuts[k], n = cuts[k + 1] - cuts[k];
            blk.resize((size_t)C * n);
            for (int c = 0; c < C; ++c) std::copy(&x[(size_t)c * N + lo], &x[(size_t)c * N + lo] + n, &blk[(size_t)c * n]);
            fft.process(blk.data(), n);
            const int nf = fft.frames();
            F += nf;
            for (int c = 0; c < C; ++c)
                for (int f = 0; f < nf; ++f) {
                    const float* m = fft.magnitudesOf(c, f);
                    mags[c].insert(mags[c].end(), m, m + bins);
                    avs[c].insert(avs[c].end(), oct.averagesOf(c, f), oct.averagesOf(c, f) + oct.nAverages);
                    pks[c].insert(pks[c].end(), oct.peaksOf(c, f), oct.peaksOf(c, f) + oct.nAverages);
                    spec[c].insert(spec[c].end(), bark.specificLoudnessOf(c, f), bark.specificLoudnessOf(c, f) + 24);
                    rel[c].insert(rel[c].end(), bark.relativeLoudnessOf(c, f), bark.relativeLoudnessOf(c, f) + 24);
                    tot[c].push_back(bark.totalLoudnessOf(c, f));
                }
        }
        int32_t h[5] = {F, oct.nAverages, refusal(C, fftSize, fftSize, x, N), refusal(C, fftSize, fftSize / 4, x, N), 0};
        const std::vector<float> quiet((size_t)C * 2 * hop, 0.f);
        fft.process(quiet.data(), 2 * hop);       // the transform and its analysers carry on after the refusals
        h[4] = fft.frames();
        FILE* fo = fopen(argv[2], "wb");
        fwrite(h, sizeof(int32_t), 5, fo);
        for (auto* v : {&mags, &avs, &pks}) for (int c = 0; c < C; ++c) put(fo, (*v)[c]);
        for (auto* v : {&spec, &rel, &tot}) for (int c = 0; c < C; ++c) put(fo, (*v)[c]);
        fclose(fo);
    } catch (const std::exception& e) { fprintf(stderr, "%s\n", e.what()); return 1; }
    return 0;
}
