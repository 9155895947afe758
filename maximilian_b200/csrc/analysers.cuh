// maxiFFTOctaveAnalyzer::calculate (src/libs/maxiFFT.cpp:264-300) and maxiBark's specificLoudness / relativeLoudness / totalLoudness
// (src/libs/maxiBark.h:63-113) on one frame, run by one warp -- included by spectral.cu for the stand-alone kernels on caller-supplied
// spectra (mxb_octave_process / mxb_bark_process). `mag` is the staged frame; the bodies convert exactly as the reference does (float
// products and sums for the octave runs, a double sum for the Bark bands).
//
// The 1024-point stream kernel's epilogue (stft_stream.cuh) performs the same operations in the same order on its magnitudes held as
// doubles, and the GPU tests hold the two paths to the same bits. It keeps its own copy: with these bodies inlined there, ptxas reports
// the same registers and spills (128; 36 B stores, 40 B loads) but schedules stft_stream_kernel<true> differently, and bench.py
// --workload spectral measured it slower on an H100 80GB HBM3 at a 700 W power limit, three interleaved runs of each: analysis_octave_bark
// 2.07-2.17 ms -> 2.20-2.22 ms, and analysis_mags_phases -- which runs no analyser -- 2.24-2.26 ms -> 2.31-2.32 ms.
#pragma once

namespace {

struct OctaveDev {
    const int* runs;           // [nruns][4]: first bin, last bin, first band, one past the last band (octave_map)
    int nruns, navg, hold;
    float decay, icpt, slope;  // peakDecayRate, linearEQIntercept, linearEQSlope
};

// The averages of one frame: one lane per run of bins. The reference's running float sum closes a run ON the first bin of the next
// averaging band, and its average goes to every band in [first band, one past the last band). Bands no run reaches keep their value.
template <class T>
__device__ __forceinline__ void octave_runs(const OctaveDev& o, const T* mag, float* avs, const int lane) {
    for (int r = lane; r < o.nruns; r += 32) {
        const int4 run = ((const int4*)o.runs)[r];
        float sum = 0.f;
        for (int b = run.x; b <= run.y; ++b)
            sum = __fadd_rn(sum, __fmul_rn((float)mag[b], __fadd_rn(o.icpt, __fmul_rn((float)b, o.slope))));
        const float av = __fdiv_rn(sum, (float)(run.y - run.x + 1));
        for (int j = run.z; j < run.w; ++j) avs[j] = av;
    }
}

// The peak hold / decay of one frame, one lane per averaging band (after octave_runs and a __syncwarp). Frame `of` of the outputs
// (each optional) receives the averages and the updated peaks.
__device__ __forceinline__ void octave_peaks(const OctaveDev& o, const float* avs, float* pks, int* hds, float* avg_out, float* peak_out,
                                             const size_t of, const int lane) {
    const int nA = o.navg;
    for (int i = lane; i < nA; i += 32) {
        const float av = avs[i];
        float pk = pks[i]; int hd = hds[i];
        if (av >= pk) { pk = av; hd = o.hold; }
        else { if (hd > 0) hd--; else pk = __fmul_rn(pk, o.decay); }
        pks[i] = pk; hds[i] = hd;
        if (avg_out) avg_out[of * nA + i] = av;
        if (peak_out) peak_out[of * nA + i] = pk;
    }
}

// maxiBark on one frame: one lane per band, double sums in bin order, libdevice pow, the max of the bands from 0 (NaN bands lose every
// `>` test, as in the reference), the total in band order by lane 0. lim: bbLimits[25] (bark_limits); bsc: 24 doubles of this warp's
// shared memory. Frame `of` of the outputs (each optional). Ends with a __syncwarp.
template <class T>
__device__ __forceinline__ void bark_frame(const int* lim, const T* mag, double* bsc, double* specific, double* relative, double* total,
                                           const size_t of, const int lane) {
    double spec = 0.0;
    if (lane < 24) {
        double sum = 0.0;
        for (int j = lim[lane]; j < lim[lane + 1]; ++j) sum = __dadd_rn(sum, (double)mag[j]);
        spec = pow(sum, 0.23);
        bsc[lane] = spec;
    }
    double mx = spec > 0.0 ? spec : 0.0;                   // `if (specific[i] > max) max = specific[i]` from max = 0
#pragma unroll
    for (int m = 16; m >= 1; m >>= 1) { const double o = __shfl_xor_sync(0xffffffffu, mx, m); mx = o > mx ? o : mx; }
    __syncwarp();
    if (lane < 24) {
        if (specific) specific[of * 24 + lane] = spec;
        if (relative) relative[of * 24 + lane] = spec / mx;
    }
    if (lane == 0 && total) {
        double t = 0.0;
        for (int i = 0; i < 24; ++i) t = __dadd_rn(t, bsc[i]);
        total[of] = t;
    }
    __syncwarp();
}

}  // namespace
