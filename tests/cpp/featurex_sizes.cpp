// The per-sample feature extractor of patch_featurex.cpp -- `if (fft.process(sample)) { oct.calculate(...); bark.specificLoudness(...); }`
// -- at any transform size, against include/maximilian_b200.hpp: an octave analyser and a maxiBark attached to the maxiFFT (at sizes
// other than 1024 the transform's process() runs them on the magnitudes it wrote), and a second pair that is NOT attached and is handed
// a spectrum made here, the magnitudes divided by the fft size (the "normalised spectrum" of the reference's signature).
//
//   featurex_sizes <in.bin> <out.bin> N fftSize
// in.bin:  N float32 samples of one channel.
// out.bin: int32 F, int32 nAverages, float32 fired[N] (1 where process() returned true), mags[F][fftSize/2],
//          attached: averages[F][nAverages], peaks[F][nAverages], float64 specific[F][24], relative[F][24], total[F],
//          not attached: float32 averages[F][nAverages], peaks[F][nAverages], float64 specific[F][24], relative[F][24], total[F].
#include <cstdio>
#include <cstdlib>
#include <vector>

#include "maximilian_b200.hpp"

template <class T> static void put(FILE* f, const std::vector<T>& v) { fwrite(v.data(), sizeof(T), v.size(), f); }

int main(int argc, char** argv) {
    if (argc != 5) { fprintf(stderr, "usage: featurex_sizes in.bin out.bin N fftSize\n"); return 2; }
    const int N = atoi(argv[3]), fftSize = atoi(argv[4]), hopSize = fftSize / 2, bins = fftSize / 2;
    vector<float> x((size_t)N);
    FILE* fi = fopen(argv[1], "rb");
    if (!fi || fread(x.data(), sizeof(float), x.size(), fi) != x.size()) { fprintf(stderr, "cannot read %s\n", argv[1]); return 1; }
    fclose(fi);
    try {
        maxiSettings::setup(48000, 2, 512);
        maxiFFT mfft;
        maxiFFTOctaveAnalyzer oct, oct2;
        maxiBark bark, bark2;
        mfft.setup(fftSize, hopSize, fftSize);
        oct.setup(48000, bins, 3);
        bark.setup(48000, fftSize);
        mfft.attach(oct); mfft.attach(bark);
        oct2.setup(48000, bins, 3);
        bark2.setup(48000, fftSize);
        for (maxiFFTOctaveAnalyzer* o : {&oct, &oct2}) { o->peakHoldTime = 2; o->peakDecayRate = 0.8f; o->linearEQIntercept = 0.9f; o->linearEQSlope = 0.01f; }

        vector<float> fired((size_t)N, 0.f), mags, avs, pks, avs2, pks2, norm((size_t)bins);
        vector<double> spec, rel, tot, spec2, rel2, tot2;
        for (int i = 0; i < N; ++i) {
            if (mfft.process(x[(size_t)i])) {
                fired[(size_t)i] = 1.f;
                vector<float>& m = mfft.getMagnitudes();
                mags.insert(mags.end(), m.begin(), m.begin() + bins);
                oct.calculate(&m[0]);
                avs.insert(avs.end(), oct.averages, oct.averages + oct.nAverages);
                pks.insert(pks.end(), oct.peaks, oct.peaks + oct.nAverages);
                const double* s = bark.specificLoudness(&m[0]); spec.insert(spec.end(), s, s + 24);
                const double* r = bark.relativeLoudness(&m[0]); rel.insert(rel.end(), r, r + 24);
                tot.push_back(bark.totalLoudness(&m[0])[0]);

                for (int b = 0; b < bins; ++b) norm[(size_t)b] = m[(size_t)b] / fftSize;
                oct2.calculate(norm.data());
                avs2.insert(avs2.end(), oct2.averages, oct2.averages + oct2.nAverages);
                pks2.insert(pks2.end(), oct2.peaks, oct2.peaks + oct2.nAverages);
                s = bark2.specificLoudness(norm.data()); spec2.insert(spec2.end(), s, s + 24);
                r = bark2.relativeLoudness(norm.data()); rel2.insert(rel2.end(), r, r + 24);
                tot2.push_back(bark2.totalLoudness(norm.data())[0]);
            }
        }
        const int32_t F = (int32_t)tot.size(), nA = oct.nAverages;
        if (oct2.nAverages != nA) { fprintf(stderr, "nAverages %d vs %d\n", oct2.nAverages, nA); return 1; }
        FILE* fo = fopen(argv[2], "wb");
        fwrite(&F, sizeof(F), 1, fo); fwrite(&nA, sizeof(nA), 1, fo);
        put(fo, fired); put(fo, mags); put(fo, avs); put(fo, pks); put(fo, spec); put(fo, rel); put(fo, tot);
        put(fo, avs2); put(fo, pks2); put(fo, spec2); put(fo, rel2); put(fo, tot2);
        fclose(fo);
    } catch (const std::exception& e) { fprintf(stderr, "%s\n", e.what()); return 1; }
    return 0;
}
