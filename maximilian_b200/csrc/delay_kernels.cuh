// K2 interface: bank kernel with a maxiDelayline stage (kernel: delay_impl.cuh; instantiations: delay_k.cu).
#pragma once

#include "bank_kernels.cuh"

namespace mxb {

constexpr int kDlShift = 4;
constexpr int kDlChunk = 1 << kDlShift;     // ring slots per chunk = time steps per staged window (16)
// the swizzle of voice v's chunk: v % 16
__host__ __device__ inline int dl_swz(size_t v) { return (int)(v & 15); }

// Ring storage is chunk-interleaved and swizzled: slot r of voice v lives at ((r / 16) * V + v) * 16 + ((r % 16) ^ (v % 16)).
// A voice's 16-slot chunk is 128 contiguous bytes (4 full sectors whatever its phase), and voices whose
// ring indices run in step -- the common case: same size, started together -- read and write one
// contiguous run of 32 * 128 B per warp and stage: ONE bulk copy (cp.async.bulk, the TMA engine) in each direction moves a
// warp's window between HBM and shared memory. The XOR with the voice index is what makes the image that lands in shared
// memory usable as it is: lane v reads slot j of its row at position j ^ (v % 16), so the 16 lanes of a half-warp hit 16
// different 8-byte bank pairs -- conflict-free without padding, which a bulk copy could not produce.
__host__ __device__ inline size_t dl_slot(size_t V, size_t v, int r) {
    return (((size_t)(r >> kDlShift)) * V + v) * kDlChunk + (size_t)((r ^ dl_swz(v)) & (kDlChunk - 1));
}
inline size_t dl_ring_doubles(size_t V, int taps) { return (size_t)((taps + kDlChunk - 1) / kDlChunk) * kDlChunk * V; }

struct DelayArgs {
    int* phase;              // maxiDelayline::phase per voice
    const int* size;         // dl() size argument per voice
    const double* feedback;
    double* ring;
    int taps;
    int from_position;       // 1: maxiDelayline::dlFromPosition
    const int* position;     // its position argument per voice
    const double* size_tv;   // optional per-sample size argument [n_frames][V] (integral values), else NULL
};

// warps the K2 grid will have for V voices: those that own at least one voice (the caller sizes the mix partials with it and
// passes it as a.W)
inline int delay_bank_warps(int V) { return (V + 31) / 32; }

// The K2 instantiations of filter family FILT (FILT_T_*); MODK: those for blocks with a per-sample oscillator frequency / filter
// cutoff. Defined in delay_k.cu, which build.py compiles once per family and MODK. outmode 0 none / 1 fp64 / 2 fp32.
template <int FILT, bool MODK>
int launch_delay_filt(const BankArgs& a, const DelayArgs& d, int osc_saw, int env, int outmode, bool mix, cudaStream_t s);

}  // namespace mxb
