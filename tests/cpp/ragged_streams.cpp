// Channels that advance independently through include/maximilian_b200.hpp: one maxiFFT of C channels fed a different number of samples
// per channel and call (maxiFFT::process(values, nSamples[])), its magnitudes / phases resynthesised by one maxiIFFT of C channels, each
// channel with its own frame count (maxiIFFT::process(mags, phases, frames[], maxFrames)). At fft size 1024 a maxiFFTOctaveAnalyzer is
// attached (fused, per channel); at other sizes a maxiBark (the fired frames packed).
//
//   ragged_streams <in.bin> <counts.bin> <out.bin> C N calls fftSize hopSize
// in.bin:     float32 x[C][N], each channel's stream.
// counts.bin: int32 counts[calls][C], the samples channel c takes in each call (the sum over calls <= N).
// out.bin:    int32 nAverages (0 without the octave analyser), then per call and channel: int32 frames(c), float32 mags[frames][bins],
//             then with the octave analyser float32 averages[frames][nAverages], peaks[frames][nAverages], else float64 totalLoudness[frames];
//             then float32 out[frames * hopSize].
#include <cstdio>
#include <cstdlib>
#include <vector>

#include "maximilian_b200.hpp"

int main(int argc, char** argv) {
    if (argc != 9) { fprintf(stderr, "usage: ragged_streams in.bin counts.bin out.bin C N calls fftSize hopSize\n"); return 2; }
    const int C = atoi(argv[4]), N = atoi(argv[5]), calls = atoi(argv[6]), fftSize = atoi(argv[7]), hopSize = atoi(argv[8]);
    vector<float> x((size_t)C * N);
    vector<int> counts((size_t)calls * C);
    FILE* fi = fopen(argv[1], "rb");
    if (!fi || fread(x.data(), sizeof(float), x.size(), fi) != x.size()) { fprintf(stderr, "cannot read %s\n", argv[1]); return 1; }
    fclose(fi);
    fi = fopen(argv[2], "rb");
    if (!fi || fread(counts.data(), sizeof(int), counts.size(), fi) != counts.size()) { fprintf(stderr, "cannot read %s\n", argv[2]); return 1; }
    fclose(fi);
    try {
        maxiSettings::setup(44100, 1, 512);
        maxiFFT fft(C);
        maxiIFFT ifft(C);
        maxiFFTOctaveAnalyzer oct;
        maxiBark bark;
        const bool octave = fftSize == 1024;
        fft.setup(fftSize, hopSize, fftSize);
        ifft.setup(fftSize, hopSize, fftSize);
        if (octave) {
            oct.setup(44100.f, fftSize / 2, 3);
            oct.peakHoldTime = 3; oct.peakDecayRate = 0.85f;
            fft.attach(oct);
        } else {
            bark.setup(44100, fftSize);
            fft.attach(bark);
        }
        const int bins = fft.getNumBins(), nA = octave ? oct.nAverages : 0;
        FILE* fo = fopen(argv[3], "wb");
        fwrite(&nA, sizeof(int), 1, fo);
        vector<size_t> off((size_t)C, 0);
        for (int k = 0; k < calls; ++k) {
            const int* cnt = &counts[(size_t)k * C];
            int pitch = 1;
            for (int c = 0; c < C; ++c) pitch = cnt[c] > pitch ? cnt[c] : pitch;
            vector<float> block((size_t)C * pitch, 0.f);
            for (int c = 0; c < C; ++c)
                for (int i = 0; i < cnt[c]; ++i) block[(size_t)c * pitch + i] = x[(size_t)c * N + off[(size_t)c] + i];
            fft.process(block.data(), cnt);
            vector<int> fr((size_t)C);
            for (int c = 0; c < C; ++c) fr[(size_t)c] = fft.frames(c);
            vector<float>& y = ifft.process(fft.getMagnitudes(), fft.getPhases(), fr.data(), fft.frameStride());
            for (int c = 0; c < C; ++c) {
                const int f = fr[(size_t)c];
                fwrite(&f, sizeof(int), 1, fo);
                if (f > 0) fwrite(fft.magnitudesOf(c, 0), sizeof(float), (size_t)f * bins, fo);
                if (octave) {
                    if (f > 0) fwrite(oct.averagesOf(c, 0), sizeof(float), (size_t)f * nA, fo);
                    if (f > 0) fwrite(oct.peaksOf(c, 0), sizeof(float), (size_t)f * nA, fo);
                } else {
                    for (int j = 0; j < f; ++j) { const double t = bark.totalLoudnessOf(c, j); fwrite(&t, sizeof(double), 1, fo); }
                }
                if (f > 0) fwrite(&y[(size_t)c * fft.frameStride() * hopSize], sizeof(float), (size_t)f * hopSize, fo);
                off[(size_t)c] += (size_t)cnt[c];
            }
        }
        fclose(fo);
    } catch (const std::exception& e) { fprintf(stderr, "%s\n", e.what()); return 1; }
    return 0;
}
