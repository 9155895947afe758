// K4s: the 1024-point streaming STFT (+ fused MFCC) kernel -- included by spectral.cu.
//
// Same arithmetic as stft_kernel (the reference's float radix-2 transform replayed butterfly for butterfly, see the
// head of spectral.cu), different schedule:
//
//   * one warp transforms TWO channels at once, frame f of channel 2k in the low half and of channel 2k+1 in the high
//     half of a 64-bit register pair: every butterfly, untangle and power step works on both frames (two scalar IEEE
//     round-to-nearest instructions per step on sm_90, which has no packed fp32). Sums of products are written
//     fma(p, 1, q) / fma(q, -1, p) with the +-1 coming from kernel arguments (opaque to the optimiser): round(p*1 + q) is
//     the separately rounded sum the reference computes, and no compiler contraction can merge the product into it.
//   * a warp walks the consecutive frames of its channel pair (pair-major order): the n - hop samples two frames share
//     are re-read from L1/L2, never from DRAM, and with several hops per call the assembly buffer (maxiFFT::buffer) is
//     read and written once per call instead of once per frame.
//   * frames are loaded straight from global memory in bit-reversed order (lane-contiguous float2 requests, 256 B per
//     request), windowed and packed in registers -- no staging pass through shared memory.
//   * the last radix-2 stage, the real-FFT untangling pass and the magnitudes run as ONE pass over shared memory: the
//     lane that owns point p also owns 256 - p, so it holds all four inputs of bins p, 256 - p, 256 + p and 512 - p.
//   * the whole MFCC stage runs on the fp64 tensor cores (mma.sync m8n8k4, SASS DMMA), 8 frames -- one 4-warp group -- at a time:
//     mel bands = [8 frames x bins] . [bins x 8 filters] per filter tile, walking only the bins the tile's filters cover (the
//     bank is banded: 377 non-zeros of 21 504), log on the accumulator fragment, then the DCT [8 x filters] . [filters x coeffs];
//     two named barriers per batch and group (magnitudes ready / mel rows ready), mel rows double-buffered.
#pragma once
#include <type_traits>

namespace {

typedef unsigned long long u64;

// Cache steering. The frames stream through (each sample is read by two consecutive frames, ~10 us apart): the second, last read
// bypasses L1 so that the few KB every frame re-reads -- the tensor-core B fragments of the mel bank and the DCT -- stay there.
// (Both reads past L1 cost more DRAM traffic: the second read then misses L2 too often.)
__device__ __forceinline__ float2 ld_stream_f2(const float* p) {
    float2 v;
    asm volatile("ld.global.L1::no_allocate.v2.f32 {%0, %1}, [%2];" : "=f"(v.x), "=f"(v.y) : "l"(p));
    return v;
}
__device__ __forceinline__ float4 ld_stream_f4(const float* p) {
    float4 v;
    asm volatile("ld.global.L1::no_allocate.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "l"(p));
    return v;
}
__device__ __forceinline__ double ld_keep_f64(const double* p) {
    double v;
    asm("ld.global.nc.L1::evict_last.f64 %0, [%1];" : "=d"(v) : "l"(p));
    return v;
}

// One m8n8k4 fp64 tensor-core step (SASS DMMA): C[8 x 8] += A[8 x 4] . B[4 x 8]; lane holds A[lane / 4][lane % 4], B[lane % 4][lane / 4],
// C[lane / 4][2 * (lane % 4) + {0, 1}].
__device__ __forceinline__ void dmma884(double& c0, double& c1, const double av, const double bv) {
    asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0, %1}, {%2}, {%3}, {%0, %1};\n" : "+d"(c0), "+d"(c1) : "d"(av), "d"(bv));
}
// C = A . B over `ksteps` k-steps: A from shared memory (this lane's element of k-step ks at ap[4 * ks]), B pre-arranged fragments in
// global memory (bfrag[32 * ks]). A single accumulator would make every step wait for the one before it AND for its own loads; here four
// accumulators take the k-steps round robin and the operands of four steps are requested together.
// The order of the fp64 additions is fixed (by k-step mod 4, then ((0 + 1) + (2 + 3))): results are reproducible from run to run.
__device__ __forceinline__ void dmma_tile(const double* __restrict__ ap, const double* __restrict__ bfrag, const int ksteps, double& c0, double& c1) {
    double acc[4][2] = {{0.0, 0.0}, {0.0, 0.0}, {0.0, 0.0}, {0.0, 0.0}};
    const int groups = ksteps >> 2;
#pragma unroll 1
    for (int g = 0; g < groups; ++g) {
        double av[4], bv[4];
#pragma unroll
        for (int i = 0; i < 4; ++i) { av[i] = ap[16 * g + 4 * i]; bv[i] = ld_keep_f64(bfrag + 128 * g + 32 * i); }
#pragma unroll
        for (int i = 0; i < 4; ++i) dmma884(acc[i][0], acc[i][1], av[i], bv[i]);
    }
    for (int ks = 4 * groups, i = 0; ks < ksteps; ++ks, ++i) {
        const double x = ap[4 * ks], y = ld_keep_f64(bfrag + 32 * ks);
        if (i == 0) dmma884(acc[0][0], acc[0][1], x, y);
        else if (i == 1) dmma884(acc[1][0], acc[1][1], x, y);
        else dmma884(acc[2][0], acc[2][1], x, y);
    }
    c0 = __dadd_rn(__dadd_rn(acc[0][0], acc[1][0]), __dadd_rn(acc[2][0], acc[3][0]));
    c1 = __dadd_rn(__dadd_rn(acc[0][1], acc[1][1]), __dadd_rn(acc[2][1], acc[3][1]));
}

// Natural logarithm of a normal, positive double, within 1 ulp of the correctly rounded value (checked against libm on 2e7
// arguments between e^-40 and e^41 and around 1). The argument reduction and the degree-14 polynomial in s = f / (2 + f) are the
// classic ones (x = 2^k (1 + f), sqrt(2)/2 < 1 + f < sqrt(2); log(1 + f) = f - f^2/2 + s (f^2/2 + R(s^2))); the quotient comes from a
// single-precision reciprocal refined twice. About 40 straight-line instructions against libdevice's ~90 with branches: two calls next
// to each other interleave. Only the mel stage uses it: its arguments are squares > 1e-12, or +inf (log(+inf) = +inf, like libm; the
// reduction below would read the exponent field of +inf as 2^1024 and return 1024 ln 2).
__device__ __forceinline__ double log_pos(double x) {
    const double x0 = x;
    int hx = __double2hiint(x);
    const int lx = __double2loint(x);
    int kexp = (hx >> 20) - 1023;
    hx &= 0x000fffff;
    const int up = (hx + 0x95f64) & 0x100000;                     // mantissa above sqrt(2): halve it, count the exponent up
    x = __hiloint2double(hx | (up ^ 0x3ff00000), lx);
    kexp += up >> 20;
    const double f = __dadd_rn(x, -1.0), d = __dadd_rn(2.0, f);
    float r0;
    asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(r0) : "f"(__double2float_rn(d)));
    double r = (double)r0;
    r = __fma_rn(r, __fma_rn(-d, r, 1.0), r);
    r = __fma_rn(r, __fma_rn(-d, r, 1.0), r);
    const double s = __dmul_rn(f, r), dk = (double)kexp;
    const double z = __dmul_rn(s, s), w = __dmul_rn(z, z);
    const double t1 = __dmul_rn(w, __fma_rn(w, __fma_rn(w, 1.531383769920937332e-01, 2.222219843214978396e-01), 3.999999999940941908e-01));
    const double t2 = __dmul_rn(z, __fma_rn(w, __fma_rn(w, __fma_rn(w, 1.479819860511658591e-01, 1.818357216161805012e-01), 2.857142874366239149e-01),
                                            6.666666666666735130e-01));
    const double R = __dadd_rn(t2, t1), hfsq = __dmul_rn(__dmul_rn(0.5, f), f);
    const double lo = __fma_rn(s, __dadd_rn(hfsq, R), __dmul_rn(dk, 1.90821492927058770002e-10));
    const double y = __dsub_rn(__dmul_rn(dk, 6.93147180369123816490e-01), __dsub_rn(__dsub_rn(hfsq, lo), f));
    return x0 == (double)INFINITY ? x0 : y;
}

__device__ __forceinline__ u64 pk2(float lo, float hi) { u64 r; asm("mov.b64 %0, {%1, %2};" : "=l"(r) : "f"(lo), "f"(hi)); return r; }
__device__ __forceinline__ void upk2(u64 v, float& lo, float& hi) { asm("mov.b64 {%0, %1}, %2;" : "=f"(lo), "=f"(hi) : "l"(v)); }
// Hopper has no packed fp32 arithmetic: each pair operation is two scalar .rn instructions on the halves of the register pair
// (the mov.b64 packing costs nothing, a 64-bit value already lives in two 32-bit registers). Same roundings as one per-half op.
__device__ __forceinline__ u64 add2(u64 a, u64 b) {
    float al, ah, bl, bh; upk2(a, al, ah); upk2(b, bl, bh);
    return pk2(__fadd_rn(al, bl), __fadd_rn(ah, bh));
}
__device__ __forceinline__ u64 sub2(u64 a, u64 b) {
    float al, ah, bl, bh; upk2(a, al, ah); upk2(b, bl, bh);
    return pk2(__fsub_rn(al, bl), __fsub_rn(ah, bh));
}
__device__ __forceinline__ u64 mul2(u64 a, u64 b) {
    float al, ah, bl, bh; upk2(a, al, ah); upk2(b, bl, bh);
    return pk2(__fmul_rn(al, bl), __fmul_rn(ah, bh));
}
__device__ __forceinline__ u64 fma2(u64 a, u64 b, u64 c) {
    float al, ah, bl, bh, cl, ch; upk2(a, al, ah); upk2(b, bl, bh); upk2(c, cl, ch);
    return pk2(__fmaf_rn(al, bl, cl), __fmaf_rn(ah, bh, ch));
}

struct Pk { u64 one, mone, half, mhalf; };        // (1,1) (-1,-1) (.5,.5) (-.5,-.5), from kernel arguments

// fft.cpp:184-192 on two frames at once; w.x = (wx, wx), w.y = (wy, wy)
__device__ __forceinline__ void butterfly2(u64& Rj, u64& Ij, u64& Rk, u64& Ik, const ulonglong2 w, const Pk& c) {
    const u64 tr = fma2(mul2(w.y, Ik), c.mone, mul2(w.x, Rk));       // round(wx*Rk - wy*Ik), both products rounded first
    const u64 ti = fma2(mul2(w.y, Rk), c.one, mul2(w.x, Ik));        // round(wx*Ik + wy*Rk)
    Rk = sub2(Rj, tr);
    Ik = sub2(Ij, ti);
    Rj = add2(Rj, tr);
    Ij = add2(Ij, ti);
}

// fft.cpp:256-272 for the pair (i, i3 = half - i) on two frames at once; w.x = (wr, wr), w.y = (wi, wi).
// NEED3: also produce the i3 side (bins above half/2).
template <bool NEED3>
__device__ __forceinline__ void untangle2(u64& Ri, u64& Ii, u64& R3, u64& I3, const ulonglong2 w, const Pk& c) {
    const u64 h1r = mul2(c.half, add2(Ri, R3));
    const u64 h1i = mul2(c.half, sub2(Ii, I3));
    const u64 h2r = mul2(c.half, add2(Ii, I3));
    const u64 h2i = mul2(c.mhalf, sub2(Ri, R3));
    const u64 a1 = mul2(w.x, h2r), a2 = mul2(w.y, h2i), a3 = mul2(w.x, h2i), a4 = mul2(w.y, h2r);
    Ri = fma2(a2, c.mone, fma2(a1, c.one, h1r));                      // (h1r + a1) - a2
    Ii = fma2(a4, c.one, fma2(a3, c.one, h1i));                       // (h1i + a3) + a4
    if (NEED3) {
        R3 = fma2(a2, c.one, fma2(a1, c.mone, h1r));                  // (h1r - a1) + a2
        I3 = fma2(a4, c.one, fma2(h1i, c.mone, a3));                  // (-h1i + a3) + a4
    }
}

constexpr int kStreamWarps = 8;        // warps per CTA = channel pairs in flight per CTA (groups of 4 warps = 8 frames per MFCC batch)
// 2 x 8 warps caps the kernel at 128 registers; on sm_90a that spills a little, yet 2 x 4 warps (no spill) is slower on the full-spectrum
// instantiation and only slightly faster on the MFCC one (DESIGN.md, K4s)
constexpr int kStreamCtasPerSm = 2;
static_assert(kStreamWarps % 4 == 0, "4-warp groups, two named barriers each");
// named barrier `id` for the 128 threads of a group; literal ids: a register id would reserve all 16 barriers
__device__ __forceinline__ void group_barrier(const int id) {
    switch (id) {
#define MXB_BAR(I) case I: asm volatile("bar.sync " #I ", 128;" ::: "memory"); break;
        MXB_BAR(1) MXB_BAR(2) MXB_BAR(3) MXB_BAR(4) MXB_BAR(5) MXB_BAR(6) MXB_BAR(7) MXB_BAR(8) MXB_BAR(9) MXB_BAR(10) MXB_BAR(11) MXB_BAR(12) MXB_BAR(13) MXB_BAR(14)
#undef MXB_BAR
        default: break;
    }
}
constexpr int kStreamN = 1024, kStreamHalf = 512;
__device__ __forceinline__ int psi16(int p) { return p + (p >> 4); }          // padded index of a 16-byte point record

struct StreamSmem { size_t off_tw, off_uw, off_win, off_mel, off_work, total; int melstride, dct_ksteps; };
__host__ __device__ inline StreamSmem stream_smem_layout(int nf) {
    StreamSmem L;
    L.off_tw = 0;                                                          // float4[512]: (wx, wx, wy, wy) at (be - 1) + n
    L.off_uw = L.off_tw + sizeof(float4) * 512;                            // float4[256]: (wr, wr, wi, wi)
    L.off_win = L.off_uw + sizeof(float4) * 256;                           // float[1024]
    // DCT k-steps in whole groups of four (dmma_tile), zero padded; row stride + 4 doubles: the rows of an A-fragment load fall on
    // distinct banks
    L.dct_ksteps = (((nf + 3) >> 2) + 3) & ~3;
    L.melstride = 4 * L.dct_ksteps + 4;
    L.off_mel = align16(L.off_win + sizeof(float) * kStreamN);             // double[2][16][melstride]
    L.off_work = align16(L.off_mel + sizeof(double) * 2 * 2 * kStreamWarps * (size_t)L.melstride);
    L.total = L.off_work + sizeof(ulonglong2) * (size_t)kStreamWarps * (kStreamHalf + kStreamHalf / 16);
    return L;
}

struct StreamArgs {
    StftArgs a;
    const float4* tw4;        // [511] forward twiddles, natural (be - 1) + n order, halves duplicated
    const float4* uw4;        // [256] untangle pairs, halves duplicated
    Pk pk;
};

__device__ __forceinline__ constexpr int brev4c(int r) { return ((r & 1) << 3) | ((r & 2) << 1) | ((r & 4) >> 1) | ((r & 8) >> 3); }

// sample i of one frame: i < split from the assembly buffer, else from the new samples
__device__ __forceinline__ float frame_sample(const float* hp, const float* ip, long long stride_t, int split, int i) {
    return i < split ? hp[i] : ip[(long long)i * stride_t];
}

// FULL = false: nothing but MFCCs leaves the kernel and the mel bank reads bins < 256 only: the upper-half outputs of the
// untangling pass and their magnitudes are never formed.
template <bool FULL>
__global__ void __launch_bounds__(kStreamWarps * 32, kStreamCtasPerSm) stft_stream_kernel(const StreamArgs sa) {
    const StftArgs& a = sa.a;
    extern __shared__ float4 smem4[];
    unsigned char* sm = (unsigned char*)smem4;
    constexpr int n = kStreamN, half = kStreamHalf;
    const int nf = a.has_mfcc ? a.mf.filters : 0;
    const StreamSmem L = stream_smem_layout(nf);
    ulonglong2* s_tw = (ulonglong2*)(sm + L.off_tw);
    ulonglong2* s_uw = (ulonglong2*)(sm + L.off_uw);
    float* s_win = (float*)(sm + L.off_win);
    double* s_mel = (double*)(sm + L.off_mel);
    const int melstride = L.melstride;
    for (int i = threadIdx.x; i < half - 1; i += blockDim.x) ((float4*)s_tw)[i] = sa.tw4[i];
    for (int i = threadIdx.x; i < half / 2; i += blockDim.x) ((float4*)s_uw)[i] = sa.uw4[i];
    for (int i = threadIdx.x; i < n; i += blockDim.x) s_win[i] = a.window[i];
    for (int i = threadIdx.x; i < 2 * 2 * kStreamWarps * melstride; i += blockDim.x) s_mel[i] = 0.0;     // K padding stays zero
    __syncthreads();

    const Pk pk = sa.pk;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int Lr = (int)(__brev((unsigned)lane) >> 27);          // bit-reversed lane: the frame samples this lane loads
    const int low4 = lane & 15, b8 = lane >> 4;
    ulonglong2* sW = (ulonglong2*)(sm + L.off_work) + (size_t)warp * (half + half / 16);
    // after the spectrum has been consumed the area holds the two frames' magnitudes as doubles, [2][512] (+ a skew of 4 doubles per
    // warp of the group: the 8 frame rows a tensor-core A fragment touches then fall into different banks)
    double* d_mag = (double*)sW + 4 * (warp & 3);

    const int C = a.C, frames = a.frames, hop = a.hop;
    const int npairs = (C + 1) >> 1;
    const int npb = (npairs + kStreamWarps - 1) / kStreamWarps;
    const bool planar = a.stride_t == 1;
    unsigned bc = 0;                                             // batches this CTA has run (mel row buffer = bc & 1)
#pragma unroll 1
    for (int pb = blockIdx.x; pb < npb; pb += gridDim.x) {
        const int pair = pb * kStreamWarps + warp;
        const int cA = 2 * pair, cB = cA + 1;
        const bool vA = cA < C, vB = cB < C;
        const int cBs = vB ? cB : cA;                            // a missing second channel re-reads the first (its results are dropped)
        bool tail_done = false;                                  // the next assembly buffer was written while loading the last frame
#pragma unroll 1
        for (int f = 0; f < frames; ++f, ++bc) {
            if (vA) {
                // ---- fft::calcFFT windowing (fft.cpp:499-505) + RealFFT even/odd packing (:238-241) + bit-reversed copy (:146-150):
                // register r <- complex sample rev4(r)*32 + rev5(lane), i.e. real samples 64*rev4(r) + 2*Lr and the next one
                const long long s0 = (long long)f * hop;
                const long long sp = (long long)a.pos0 - s0;
                const int split = sp < 0 ? 0 : (sp > n ? n : (int)sp);
                const float* hpA = a.hist + (size_t)cA * n + s0;
                const float* hpB = a.hist + (size_t)cBs * n + s0;
                const float* ipA = a.in + (long long)cA * a.stride_c + (s0 - a.pos0) * a.stride_t;
                const float* ipB = a.in + (long long)cBs * a.stride_c + (s0 - a.pos0) * a.stride_t;
                u64 R[16], I[16];
                // fast path: unit sample stride, 8-byte aligned rows, and a buffer/new-sample boundary on a multiple of 64 samples
                // (then all lanes of a request read the same source: the steady state of a stream fed whole hops)
                const bool vec = planar && (split & 63) == 0 &&
                                 ((((uintptr_t)hpA) | ((uintptr_t)hpB) | ((uintptr_t)ipA) | ((uintptr_t)ipB)) & 7) == 0;
                if (vec) {
                    const float* wl = s_win + 2 * Lr;
                    const float *hA = hpA + 2 * Lr, *hB = hpB + 2 * Lr, *iA = ipA + 2 * Lr, *iB = ipB + 2 * Lr;
                    // QS = split / 64 known at compile time (8: the steady state of hop 512; 0: all new; 16: all history) turns the
                    // choice of source into straight-line code; any other boundary selects per request (warp-uniform predicate)
                    // warp-uniform: this is the last frame and the unconsumed tail lies inside it (whole hops were fed)
                    const bool tail_here = f == frames - 1 && a.newpos > 0 && a.newpos <= n - hop && ((hop | a.newpos) & 1) == 0;
                    tail_done = tail_here;
                    auto load = [&](auto QS) {
                        constexpr int qs = decltype(QS)::value;
#pragma unroll
                        for (int g = 0; g < 2; ++g) {          // two groups of eight requests per channel: 32 raw values in flight
                            float2 xa[8], xb[8];
#pragma unroll
                            for (int k = 0; k < 8; ++k) {
                                const int r = 8 * g + k;
                                const bool fromhist = qs >= 0 ? brev4c(r) < qs : 64 * brev4c(r) < split;
                                // odd r = the upper half of the frame: the next frame reads it again (cached normally); even r = the lower
                                // half, read for the last time at the usual hop of n/2 (not kept in L1)
                                if (r & 1) {
                                    xa[k] = *(const float2*)((fromhist ? hA : iA) + 64 * brev4c(r));
                                    xb[k] = *(const float2*)((fromhist ? hB : iB) + 64 * brev4c(r));
                                } else {
                                    xa[k] = ld_stream_f2((fromhist ? hA : iA) + 64 * brev4c(r));
                                    xb[k] = ld_stream_f2((fromhist ? hB : iB) + 64 * brev4c(r));
                                }
                            }
                            if (tail_here) {
                                // the last frame's samples from `hop` on ARE the next assembly buffer (maxiFFT.cpp:85-87): stored from the
                                // registers they were just loaded into, not read again after the transform
#pragma unroll
                                for (int k = 0; k < 8; ++k) {
                                    const int idx = 64 * brev4c(8 * g + k) + 2 * Lr - hop;
                                    if (idx >= 0 && idx < a.newpos) {
                                        __stcs((float2*)(a.next + (size_t)cA * n + idx), xa[k]);
                                        if (vB) __stcs((float2*)(a.next + (size_t)cB * n + idx), xb[k]);
                                    }
                                }
                            }
#pragma unroll
                            for (int k = 0; k < 8; ++k) {
                                const int r = 8 * g + k;
                                const float2 w = *(const float2*)(wl + 64 * brev4c(r));
                                R[r] = pk2(__fmul_rn(xa[k].x, w.x), __fmul_rn(xb[k].x, w.x));
                                I[r] = pk2(__fmul_rn(xa[k].y, w.y), __fmul_rn(xb[k].y, w.y));
                            }
                        }
                    };
                    switch (split >> 6) {
                        case 8: load(std::integral_constant<int, 8>()); break;
                        case 0: load(std::integral_constant<int, 0>()); break;
                        case 16: load(std::integral_constant<int, 16>()); break;
                        default: load(std::integral_constant<int, -1>()); break;
                    }
                } else {
#pragma unroll
                    for (int r = 0; r < 16; ++r) {
                        const int i = 64 * brev4c(r) + 2 * Lr;
                        const float w0 = s_win[i], w1 = s_win[i + 1];
                        R[r] = pk2(__fmul_rn(frame_sample(hpA, ipA, a.stride_t, split, i), w0), __fmul_rn(frame_sample(hpB, ipB, a.stride_t, split, i), w0));
                        I[r] = pk2(__fmul_rn(frame_sample(hpA, ipA, a.stride_t, split, i + 1), w1), __fmul_rn(frame_sample(hpB, ipB, a.stride_t, split, i + 1), w1));
                    }
                }
                if (planar && f + 2 < frames) {
                    // the new samples of the frame after next, one 128-byte line per lane (16 lanes per channel = hop 512), into L2
                    const float* pfa = (lane < 16 ? ipA : ipB) + 2 * hop + (n - hop) + (lane & 15) * 32;
                    if ((lane & 15) * 32 < hop) asm volatile("prefetch.global.L2 [%0];" :: "l"(pfa));
                }
                // ---- FFT() stages with BlockEnd 1, 2, 4, 8: lane-local on 16 consecutive points ----
                {
                    int off = 0;
#pragma unroll
                    for (int be = 1; be < 16; be <<= 1) {
#pragma unroll
                        for (int blk = 0; blk < 16; blk += 2 * be)
#pragma unroll
                            for (int q = 0; q < be; ++q) butterfly2(R[blk + q], I[blk + q], R[blk + q + be], I[blk + q + be], s_tw[off + q], pk);
                        off += be;
                    }
                }
                // transpose: point lane*16 + r -> (lane >> 4)*256 + r*16 + (lane & 15)
#pragma unroll
                for (int r = 0; r < 16; ++r) sW[psi16(lane * 16 + r)] = make_ulonglong2(R[r], I[r]);
                __syncwarp();
#pragma unroll
                for (int r = 0; r < 16; ++r) { const ulonglong2 v = sW[psi16(b8 * 256 + r * 16 + low4)]; R[r] = v.x; I[r] = v.y; }
                __syncwarp();
                // ---- stages with BlockEnd 16, 32, 64, 128: partner register r | m, twiddle n = (r & (m - 1))*16 + low4 ----
#pragma unroll
                for (int m = 1; m < 16; m <<= 1) {
                    const ulonglong2* t = s_tw + (16 * m - 1) + low4;
#pragma unroll
                    for (int r = 0; r < 16; ++r) {
                        if (r & m) continue;
                        butterfly2(R[r], I[r], R[r | m], I[r | m], t[(r & (m - 1)) * 16], pk);
                    }
                }
#pragma unroll
                for (int r = 0; r < 16; ++r) sW[psi16(b8 * 256 + r * 16 + low4)] = make_ulonglong2(R[r], I[r]);
                __syncwarp();
                // ---- last stage (BlockEnd 256) + RealFFT untangling (fft.cpp:256-275) + cartToPol (:507-515), one pass ----
                // item p: butterflies (p, p+256) and (256-p, 512-p) give X[p], X[p+256], X[256-p], X[512-p]: the inputs of
                // untangle pairs (p, 512-p) and (256-p, 256+p). Lane 0's first item is the odd one out: butterflies (128, 384)
                // and (0, 256), pair (128, 384), DC/Nyquist packing of bin 0, bin 256 left as it is (N/4 is never untangled).
                const size_t oA = ((size_t)cA * a.max_frames + f) * half, oB = ((size_t)cBs * a.max_frames + f) * half;
                float mg[4][4];                                  // [item][A bin1, B bin1, A bin3, B bin3] (+ FULL: written out directly)
                // psi16(32*it + lane) = lane + (lane >> 4) + 34*it;  psi16(256 - 32*it - lane) = u + (u >> 4) + 238 - 34*it with u = 32 - lane
                const int ia0 = lane + (lane >> 4), iq0 = (32 - lane) + ((32 - lane) >> 4) + 238;
                float fgmA = 0.f, famA = 0.f, fxA = 0.f, fgmB = 0.f, famB = 0.f, fxB = 0.f;
                const bool feat = FULL && (a.flatness != nullptr || a.centroid != nullptr);
#pragma unroll
                for (int it = 0; it < 4; ++it) {
                    const int p = it * 32 + lane;
                    const bool special = it == 0 && lane == 0;
                    const int pa = special ? 128 : p, pq = special ? 0 : 256 - p;
                    const int ia = (it == 0 && special) ? psi16(128) : ia0 + 34 * it, iq = (it == 0 && special) ? 0 : iq0 - 34 * it;
                    ulonglong2 Aj = sW[ia], Ak = sW[ia + 272], Bj = sW[iq], Bk = sW[iq + 272];
                    butterfly2(Aj.x, Aj.y, Ak.x, Ak.y, s_tw[255 + pa], pk);
                    butterfly2(Bj.x, Bj.y, Bk.x, Bk.y, s_tw[255 + pq], pk);
                    // pair 1: (i, i3) = (pa, special ? 384 : 512 - p); pair 2 (generic items only): (256 - p, 256 + p)
                    u64 R3 = special ? Ak.x : Bk.x, I3 = special ? Ak.y : Bk.y;
                    untangle2<FULL>(Aj.x, Aj.y, R3, I3, s_uw[pa], pk);
                    u64 U2r = Bj.x, U2i = Bj.y, U23r = Ak.x, U23i = Ak.y;
                    // MFCC-only: pair 2 feeds bin 256 - p alone; when no lane of this item row has it below the mel bank's last
                    // bin the pair is skipped (lane 0's bin 0 is patched in below)
                    const bool skip2 = !FULL && 225 - 32 * it >= a.mf.maxbin;
                    if (!skip2) untangle2<FULL>(U2r, U2i, U23r, U23i, s_uw[special ? 1 : pq], pk);
                    if (it == 0) {      // lane 0: bin 0 = (re + im, re - im) of X[0] (fft.cpp:274-275), bin 256 = X[256]
                        const u64 dcr = add2(Bj.x, Bj.y), dci = sub2(Bj.x, Bj.y);
                        U2r = special ? dcr : U2r; U2i = special ? dci : U2i;
                        U23r = special ? Bk.x : U23r; U23i = special ? Bk.y : U23i;
                    }
                    // bins: b1 <- pair 1 i side, b2 <- pair 1 i3 side, b3 <- pair 2 i side, b4 <- pair 2 i3 side
                    const int b1 = pa, b3 = pq;
                    {
                        float pA, pB;
                        upk2(fma2(mul2(Aj.x, Aj.x), pk.one, mul2(Aj.y, Aj.y)), pA, pB);
                        mg[it][0] = sqrtf(pA); mg[it][1] = sqrtf(pB);
                        upk2(fma2(mul2(U2r, U2r), pk.one, mul2(U2i, U2i)), pA, pB);
                        mg[it][2] = sqrtf(pA); mg[it][3] = sqrtf(pB);
                    }
                    if (FULL) {
                        const int b2 = special ? 384 : 512 - p, b4 = special ? 256 : 256 + p;
                        float m2A, m2B, m4A, m4B;
                        {
                            float pA, pB;
                            upk2(fma2(mul2(R3, R3), pk.one, mul2(I3, I3)), pA, pB);
                            m2A = sqrtf(pA); m2B = sqrtf(pB);
                            upk2(fma2(mul2(U23r, U23r), pk.one, mul2(U23i, U23i)), pA, pB);
                            m4A = sqrtf(pA); m4B = sqrtf(pB);
                        }
                        const int bb[4] = {b1, b2, b3, b4};
                        const u64 re[4] = {Aj.x, R3, U2r, U23r}, im[4] = {Aj.y, I3, U2i, U23i};
                        const float mA[4] = {mg[it][0], m2A, mg[it][2], m4A}, mB[4] = {mg[it][1], m2B, mg[it][3], m4B};
#pragma unroll
                        for (int k = 0; k < 4; ++k) {
                            float reA, reB, imA, imB;
                            upk2(re[k], reA, reB); upk2(im[k], imA, imB);
                            const int b = bb[k];
                            if (a.re) { a.re[oA + b] = reA; if (vB) a.re[oB + b] = reB; }
                            if (a.im) { a.im[oA + b] = imA; if (vB) a.im[oB + b] = imB; }
                            if (a.mags) { a.mags[oA + b] = mA[k]; if (vB) a.mags[oB + b] = mB[k]; }
                            if (a.phases) { a.phases[oA + b] = atan2f(imA, reA); if (vB) a.phases[oB + b] = atan2f(imB, reB); }
                            // fft::convToDB, src/libs/fft.cpp:526-534: float log10 of (mag + 1), scaled in double, stored as float
                            if (a.mags_db) {
                                a.mags_db[oA + b] = (double)mA[k] < 0.000001 ? 0.f : (float)(20.0 * (double)log10f(__fadd_rn(mA[k], 1.f)));
                                if (vB) a.mags_db[oB + b] = (double)mB[k] < 0.000001 ? 0.f : (float)(20.0 * (double)log10f(__fadd_rn(mB[k], 1.f)));
                            }
                            if (feat) {     // maxiFFT::spectralFlatness / spectralCentroid, src/libs/maxiFFT.cpp:113-132 (lane-strided partial sums)
                                if (mA[k] != 0.f) fgmA = __fadd_rn(fgmA, logf(mA[k]));
                                famA = __fadd_rn(famA, mA[k]); fxA = __fadd_rn(fxA, __fmul_rn(fabsf(mA[k]), (float)b));
                                if (mB[k] != 0.f) fgmB = __fadd_rn(fgmB, logf(mB[k]));
                                famB = __fadd_rn(famB, mB[k]); fxB = __fadd_rn(fxB, __fmul_rn(fabsf(mB[k]), (float)b));
                            }
                        }
                        // the mel stage may read any bin: all four magnitudes go to shared memory below
                        mg[it][0] = mA[0]; mg[it][1] = mB[0]; mg[it][2] = mA[2]; mg[it][3] = mB[2];
                        // (b2 / b4 magnitudes are parked in the untangle outputs' registers)
                        Ak.x = pk2(m2A, m2B); Ak.y = pk2(m4A, m4B);
                        // keep them for the write after the pass
                        R[it] = Ak.x; I[it] = Ak.y;
                    }
                }
                __syncwarp();                                    // every lane has read its points: the area becomes d_mag[2][512]
#pragma unroll
                for (int it = 0; it < 4; ++it) {
                    const int p = it * 32 + lane;
                    const bool special = it == 0 && lane == 0;
                    const int b1 = special ? 128 : p, b3 = special ? 0 : 256 - p;
                    d_mag[b1] = (double)mg[it][0]; d_mag[half + b1] = (double)mg[it][1];
                    d_mag[b3] = (double)mg[it][2]; d_mag[half + b3] = (double)mg[it][3];
                    if (FULL) {
                        const int b2 = special ? 384 : 512 - p, b4 = special ? 256 : 256 + p;
                        float x, y;
                        upk2(R[it], x, y); d_mag[b2] = (double)x; d_mag[half + b2] = (double)y;
                        upk2(I[it], x, y); d_mag[b4] = (double)x; d_mag[half + b4] = (double)y;
                    }
                }
                if (feat) {
#pragma unroll
                    for (int m = 16; m >= 1; m >>= 1) {
                        fgmA = __fadd_rn(fgmA, __shfl_xor_sync(0xffffffffu, fgmA, m)); famA = __fadd_rn(famA, __shfl_xor_sync(0xffffffffu, famA, m));
                        fxA = __fadd_rn(fxA, __shfl_xor_sync(0xffffffffu, fxA, m));
                        fgmB = __fadd_rn(fgmB, __shfl_xor_sync(0xffffffffu, fgmB, m)); famB = __fadd_rn(famB, __shfl_xor_sync(0xffffffffu, famB, m));
                        fxB = __fadd_rn(fxB, __shfl_xor_sync(0xffffffffu, fxB, m));
                    }
                    if (lane == 0) {
                        const size_t ofA = (size_t)cA * a.max_frames + f, ofB = (size_t)cBs * a.max_frames + f;
                        if (a.flatness) {
                            a.flatness[ofA] = (famA / (float)half) != 0.f ? expf(fgmA / (float)half) / (famA / (float)half) : 0.f;
                            if (vB) a.flatness[ofB] = (famB / (float)half) != 0.f ? expf(fgmB / (float)half) / (famB / (float)half) : 0.f;
                        }
                        if (a.centroid) {
                            a.centroid[ofA] = famA != 0.f ? __fmul_rn(fxA / famA, a.bin_hz) : 0.f;
                            if (vB) a.centroid[ofB] = famB != 0.f ? __fmul_rn(fxB / famB, a.bin_hz) : 0.f;
                        }
                    }
                }
                __syncwarp();
                if (FULL && (a.oct_nruns > 0 || a.bark_lim != nullptr)) {
                    // ---- maxiFFTOctaveAnalyzer::calculate (maxiFFT.cpp:264-300) and maxiBark (maxiBark.h:63-113) on the magnitudes
                    // still in shared memory. Octave: one lane per run of bins (the reference's running float sum closes a run ON the
                    // first bin of the next averaging band), then one lane per averaging band for the peak-hold logic; the bands'
                    // averages / peaks / hold counters are per-channel state carried from frame to frame in HBM (this warp walks
                    // the channel's frames in order). Bark: one lane per band, double sums in bin order, pow, max, total.
                    double* bsc = (double*)sW + 1040;                         // 24 doubles of scratch behind d_mag[2][512] (+ skew)
#pragma unroll 1
                    for (int fr = 0; fr < 2; ++fr) {
                        const int c = fr ? cB : cA;
                        if (c >= C) break;
                        const double* mag = d_mag + fr * half;                // floats stored as doubles: the conversions back are exact
                        const size_t of = (size_t)c * a.max_frames + f;
                        if (a.oct_nruns > 0) {
                            const int nA = a.oct_navg;
                            float* avs = a.oct_avg_state + (size_t)c * nA; float* pks = a.oct_peak_state + (size_t)c * nA; int* hds = a.oct_hold_state + (size_t)c * nA;
                            for (int r = lane; r < a.oct_nruns; r += 32) {
                                const int4 run = ((const int4*)a.oct_runs)[r];          // first bin, last bin, first band, one past the last band
                                float sum = 0.f;
                                for (int b = run.x; b <= run.y; ++b)
                                    sum = __fadd_rn(sum, __fmul_rn((float)mag[b], __fadd_rn(a.oct_icpt, __fmul_rn((float)b, a.oct_slope))));
                                const float av = __fdiv_rn(sum, (float)(run.y - run.x + 1));
                                for (int j = run.z; j < run.w; ++j) avs[j] = av;
                            }
                            __syncwarp();
                            for (int i = lane; i < nA; i += 32) {
                                const float av = avs[i];
                                float pk = pks[i]; int hd = hds[i];
                                if (av >= pk) { pk = av; hd = a.oct_hold; }
                                else { if (hd > 0) hd--; else pk = __fmul_rn(pk, a.oct_decay); }
                                pks[i] = pk; hds[i] = hd;
                                if (a.oct_avg_out) a.oct_avg_out[of * nA + i] = av;
                                if (a.oct_peak_out) a.oct_peak_out[of * nA + i] = pk;
                            }
                            __syncwarp();
                        }
                        if (a.bark_lim != nullptr) {
                            double spec = 0.0;
                            if (lane < 24) {
                                double sum = 0.0;
                                for (int j = a.bark_lim[lane]; j < a.bark_lim[lane + 1]; ++j) sum = __dadd_rn(sum, mag[j]);
                                spec = pow(sum, 0.23);
                                bsc[lane] = spec;
                            }
                            double mx = spec > 0.0 ? spec : 0.0;                   // `if (specific[i] > max) max = specific[i]` from max = 0
#pragma unroll
                            for (int m = 16; m >= 1; m >>= 1) { const double o = __shfl_xor_sync(0xffffffffu, mx, m); mx = o > mx ? o : mx; }
                            __syncwarp();
                            if (lane < 24) {
                                if (a.bark_specific) a.bark_specific[of * 24 + lane] = spec;
                                if (a.bark_relative) a.bark_relative[of * 24 + lane] = spec / mx;
                            }
                            if (lane == 0 && a.bark_total) {
                                double t = 0.0;
                                for (int i = 0; i < 24; ++i) t = __dadd_rn(t, bsc[i]);
                                a.bark_total[of] = t;
                            }
                            __syncwarp();
                        }
                    }
                }
                __syncwarp();
            } else if (a.has_mfcc) {
                for (int k = lane; k < 2 * half; k += 32) d_mag[k] = 0.0;     // a warp without a channel pair contributes silent frames
                __syncwarp();
            }
            if (a.has_mfcc) {
                // ---- maxiMFCC::mfcc (maxiMFCC.h:77-111, maxiMFCC.cpp:48-66) for the 8 frames of this 4-warp group, on the fp64 tensor
                // cores (mma.sync m8n8k4, SASS DMMA). Frame row r of the group = warp r/2, channel A / B = r%2.
                //   mel:  per tile of 8 filters  C[8 x 8] = mags[8 x bins] . W[bins x 8]  over the bins the tile's filters cover
                //         (k-steps of 4 bins; B fragments pre-arranged per (tile, k-step, lane), zero outside the bands), then the
                //         gate and log on the accumulator fragment: melBands = sum > 1e-6 ? log(sum^2) : 0
                //   DCT:  per tile of 8 coefficients  C[8 x 8] = melBands[8 x filters] . D[filters x 8], / numCoeffs
                // The tensor core adds in its own order: results agree with the reference's sequential sums to fp64 reassociation
                // (~1e-15 relative; asserted at 1e-9). Two named barriers per batch and group; the mel rows are double-buffered.
                const int grp = warp >> 2, wg = warp & 3;
                const int row = lane >> 2, kk = lane & 3;
                // Mel tiles of this warp. Whole tiles go round robin from the top (the widest bands first); each costs two logarithms
                // per lane, the expensive part. A last round of one or two tiles is shared by halves -- two warps run the (narrow)
                // tile and each takes the logarithm of one accumulator -- so that 42 filters (six tiles) cost every warp three.
                const int mel_nt = a.mf.mel_ntiles, mel_rem = mel_nt & 3;
                const bool halves = mel_rem == 1 || mel_rem == 2;
                int nt = mel_nt - 1 - wg;                                           // first tile: its descriptor (fragment offset, first bin,
                int4 tile = make_int4(0, 0, 0, 0);                                  // k-steps) is requested before the wait
                if (nt >= 0) tile = __ldg((const int4*)a.mf.mel_tiles + nt);
                group_barrier(1 + grp);                                             // the group's 8 magnitude rows are in shared memory
                double* melbuf = s_mel + (size_t)(bc & 1) * 2 * kStreamWarps * melstride;
                {
                    const double* amag = (const double*)((ulonglong2*)(sm + L.off_work) + (size_t)(4 * grp + (row >> 1)) * (half + half / 16)) +
                                         4 * (row >> 1) + (row & 1) * half + kk;      // row r: warp 4*grp + r/2 (skew 4*(r/2)), frame r%2
                    double* mr = melbuf + (size_t)(8 * grp + row) * melstride;
                    const int whole_lo = halves ? mel_rem : 0;                         // tiles below this index are shared by halves
                    while (nt >= whole_lo) {
                        const int ntn = nt - 4;
                        int4 tilen = tile;
                        if (ntn >= 0) tilen = __ldg((const int4*)a.mf.mel_tiles + ntn);   // the next descriptor travels during this tile
                        double c0, c1;
                        dmma_tile(amag + tile.y, a.mf.melf + (size_t)tile.x * 32 + lane, tile.z, c0, c1);
                        const double l0 = log_pos(__dmul_rn(c0, c0)), l1 = log_pos(__dmul_rn(c1, c1));
                        const int f0 = nt * 8 + 2 * kk;
                        if (f0 < nf) mr[f0] = c0 > 0.000001 ? l0 : 0.0;                // melBands = sum > 1e-6 ? log(sum^2) : 0 (maxiMFCC.cpp:64)
                        if (f0 + 1 < nf) mr[f0 + 1] = c1 > 0.000001 ? l1 : 0.0;
                        nt = ntn; tile = tilen;
                    }
                    if (halves) {
                        // rem 2: tile 1 -> warps 0, 1; tile 0 -> warps 2, 3.  rem 1: tile 0 -> warps 0, 1
                        const int ht = mel_rem == 2 ? 1 - (wg >> 1) : (wg < 2 ? 0 : -1);
                        if (ht >= 0) {
                            const int4 th = __ldg((const int4*)a.mf.mel_tiles + ht);
                            double c0, c1;
                            dmma_tile(amag + th.y, a.mf.melf + (size_t)th.x * 32 + lane, th.z, c0, c1);
                            const double c = (wg & 1) ? c1 : c0;
                            const double l = log_pos(__dmul_rn(c, c));
                            const int fi = ht * 8 + 2 * kk + (wg & 1);
                            if (fi < nf) mr[fi] = c > 0.000001 ? l : 0.0;
                        }
                    }
                }
                group_barrier(1 + kStreamWarps / 4 + grp);                          // the group's 8 mel rows are complete, its magnitudes consumed
                const double* arow = melbuf + (size_t)(8 * grp + row) * melstride + kk;
                const int ntiles = (a.mf.coeffs + 7) >> 3, ksteps = L.dct_ksteps;
                const double ncinv = 1.0 / (double)(unsigned)a.mf.coeffs;          // dct(): `/ numCoeffs` (maxiMFCC.h:108-110) as one multiply, <= 1 ulp apart
                for (int nt = 3 - wg; nt < ntiles; nt += 4) {                       // warps 3, 2 first: they had the narrowest mel tiles
                    double c0, c1;
                    dmma_tile(arow, a.mf.dctf + (size_t)nt * ksteps * 32 + lane, ksteps, c0, c1);   // columns >= filters are zero
                    const int fi = 8 * grp + row;                // frame of the CTA's batch: warp fi >> 1, channel A / B = fi & 1
                    const int ch = 2 * (pb * kStreamWarps + (fi >> 1)) + (fi & 1);
                    if (ch < C) {
                        double* o = a.coeffs + ((size_t)ch * a.max_frames + f) * a.mf.coeffs;
                        const int cc = nt * 8 + 2 * kk;
                        if (cc < a.mf.coeffs) o[cc] = __dmul_rn(c0, ncinv);
                        if (cc + 1 < a.mf.coeffs) o[cc + 1] = __dmul_rn(c1, ncinv);
                    }
                }
            }
        }
        // ---- the channels' next assembly buffers: the unconsumed tail of (buffer ++ new samples), maxiFFT.cpp:85-87 applied
        // `frames` times. It goes to the OTHER buffer (double-buffered across calls). ----
        if (vA && a.newpos > 0 && !tail_done) {
            const long long consumed = (long long)frames * hop;
#pragma unroll 1
            for (int k = 0; k < 2; ++k) {
                const int c = k ? cB : cA;
                if (c >= C) break;
                const float* hsrc = a.hist + (size_t)c * n;
                const float* isrc = a.in + (long long)c * a.stride_c;
                float* nx = a.next + (size_t)c * n;
                const long long fromin = consumed - a.pos0;               // first new-sample index of the tail when none of it is history
                if (planar && fromin >= 0 && (a.newpos & 3) == 0 && ((((uintptr_t)(isrc + fromin)) | ((uintptr_t)nx)) & 15) == 0) {
                    for (int i = 4 * lane; i < a.newpos; i += 128) __stcs((float4*)(nx + i), ld_stream_f4(isrc + fromin + i));
                } else {
                    for (int i = lane; i < a.newpos; i += 32) {
                        const long long s = consumed + i;
                        nx[i] = s < a.pos0 ? hsrc[s] : isrc[(s - a.pos0) * a.stride_t];
                    }
                }
            }
        }
    }
}

// FULL = false: nothing but MFCCs leaves the kernel and the mel bank reads bins < 256 only: the upper-half outputs of the
// untangling pass and their magnitudes are never formed.
// stft_stream_kernel's transform for stft_stream_ragged_kernel (RAGGED = true; stft_stream_kernel keeps its own copy, so that its code
// stays the one measured; the RAGGED ? : selections mark where the two differ): every channel has its own frame count and buffer
// positions. A warp walks the longer of its two channels -- with the MFCC, the longest of its 4-warp group, whose named barriers need
// every warp of the group at each frame -- and a half past its channel's last frame computes on zeros and stores nothing (its octave
// state does not advance).
template <bool FULL, bool RAGGED>
__device__ __forceinline__ void stft_stream_body(const StreamArgs sa, const RaggedDev rg) {
    const StftArgs& a = sa.a;
    extern __shared__ float4 smem4[];
    unsigned char* sm = (unsigned char*)smem4;
    constexpr int n = kStreamN, half = kStreamHalf;
    const int nf = a.has_mfcc ? a.mf.filters : 0;
    const StreamSmem L = stream_smem_layout(nf);
    ulonglong2* s_tw = (ulonglong2*)(sm + L.off_tw);
    ulonglong2* s_uw = (ulonglong2*)(sm + L.off_uw);
    float* s_win = (float*)(sm + L.off_win);
    double* s_mel = (double*)(sm + L.off_mel);
    const int melstride = L.melstride;
    for (int i = threadIdx.x; i < half - 1; i += blockDim.x) ((float4*)s_tw)[i] = sa.tw4[i];
    for (int i = threadIdx.x; i < half / 2; i += blockDim.x) ((float4*)s_uw)[i] = sa.uw4[i];
    for (int i = threadIdx.x; i < n; i += blockDim.x) s_win[i] = a.window[i];
    for (int i = threadIdx.x; i < 2 * 2 * kStreamWarps * melstride; i += blockDim.x) s_mel[i] = 0.0;     // K padding stays zero
    __syncthreads();

    const Pk pk = sa.pk;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int Lr = (int)(__brev((unsigned)lane) >> 27);          // bit-reversed lane: the frame samples this lane loads
    const int low4 = lane & 15, b8 = lane >> 4;
    ulonglong2* sW = (ulonglong2*)(sm + L.off_work) + (size_t)warp * (half + half / 16);
    // after the spectrum has been consumed the area holds the two frames' magnitudes as doubles, [2][512] (+ a skew of 4 doubles per
    // warp of the group: the 8 frame rows a tensor-core A fragment touches then fall into different banks)
    double* d_mag = (double*)sW + 4 * (warp & 3);

    const int C = a.C, frames = a.frames, hop = a.hop;
    const int npairs = (C + 1) >> 1;
    const int npb = (npairs + kStreamWarps - 1) / kStreamWarps;
    const bool planar = a.stride_t == 1;
    unsigned bc = 0;                                             // batches this CTA has run (mel row buffer = bc & 1)
#pragma unroll 1
    for (int pb = blockIdx.x; pb < npb; pb += gridDim.x) {
        const int pair = pb * kStreamWarps + warp;
        const int cA = 2 * pair, cB = cA + 1;
        const bool vA = cA < C, vB = cB < C;
        const int cBs = vB ? cB : cA;                            // a missing second channel re-reads the first (its results are dropped)
        bool tail_done = false;                                  // the next assembly buffer was written while loading the last frame
        // the two channels' frame counts and buffer positions, and the frames this warp walks
        int frA = frames, frB = frames, posA = a.pos0, posB = a.pos0, walk = frames;
        if constexpr (RAGGED) {
            frA = vA ? ragged_frames(rg, cA) : 0; frB = vB ? ragged_frames(rg, cB) : 0;
            posA = vA ? __ldg(rg.pos0 + cA) : 0; posB = vB ? __ldg(rg.pos0 + cB) : posA;
            walk = max(frA, frB);
            if (a.has_mfcc) {
                const int g0 = 2 * (pb * kStreamWarps + 4 * (warp >> 2));         // first channel of this warp's group
                for (int k = 0; k < 8 && g0 + k < C; ++k) walk = max(walk, ragged_frames(rg, g0 + k));
            }
        }
#pragma unroll 1
        for (int f = 0; f < walk; ++f, ++bc) {
            const bool liveA = RAGGED ? f < frA : true;          // the halves that store this frame
            const bool liveB = RAGGED ? (vB && f < frB) : vB;
            if (RAGGED ? (liveA || liveB) : vA) {
                // ---- fft::calcFFT windowing (fft.cpp:499-505) + RealFFT even/odd packing (:238-241) + bit-reversed copy (:146-150):
                // register r <- complex sample rev4(r)*32 + rev5(lane), i.e. real samples 64*rev4(r) + 2*Lr and the next one
                const long long s0 = (long long)f * hop;
                const long long sp = (long long)(RAGGED ? posA : a.pos0) - s0;
                const int split = sp < 0 ? 0 : (sp > n ? n : (int)sp);
                const float* hpA = a.hist + (size_t)cA * n + s0;
                const float* hpB = a.hist + (size_t)cBs * n + s0;
                const float* ipA = a.in + (long long)cA * a.stride_c + (s0 - (RAGGED ? posA : a.pos0)) * a.stride_t;
                const float* ipB = a.in + (long long)cBs * a.stride_c + (s0 - (RAGGED ? posB : a.pos0)) * a.stride_t;
                u64 R[16], I[16];
                // the two channels' buffer / new-sample boundaries differ: each lane picks its source. float2 requests where every
                // lane's two samples come from one source and the rows are 8-byte aligned, else one sample at a time
                const long long spB = (long long)posB - s0;
                const int splitB = spB < 0 ? 0 : (spB > n ? n : (int)spB);
                const bool vec2 = planar && ((split | splitB) & 1) == 0 &&
                                  ((((uintptr_t)hpA) | ((uintptr_t)hpB) | ((uintptr_t)ipA) | ((uintptr_t)ipB)) & 7) == 0;
#pragma unroll
                for (int r = 0; r < 16; ++r) {
                    const int i = 64 * brev4c(r) + 2 * Lr;
                    const float2 w = *(const float2*)(s_win + i);
                    float2 xa = make_float2(0.f, 0.f), xb = make_float2(0.f, 0.f);
                    if (vec2) {
                        if (liveA) xa = *(const float2*)((i < split ? hpA : ipA) + i);
                        if (liveB) xb = *(const float2*)((i < splitB ? hpB : ipB) + i);
                    } else {
                        if (liveA) xa = make_float2(frame_sample(hpA, ipA, a.stride_t, split, i), frame_sample(hpA, ipA, a.stride_t, split, i + 1));
                        if (liveB) xb = make_float2(frame_sample(hpB, ipB, a.stride_t, splitB, i), frame_sample(hpB, ipB, a.stride_t, splitB, i + 1));
                    }
                    R[r] = pk2(__fmul_rn(xa.x, w.x), __fmul_rn(xb.x, w.x));
                    I[r] = pk2(__fmul_rn(xa.y, w.y), __fmul_rn(xb.y, w.y));
                }
                if (planar && (RAGGED ? (f + 2 < frA && (!vB || f + 2 < frB)) : f + 2 < frames)) {
                    // the new samples of the frame after next, one 128-byte line per lane (16 lanes per channel = hop 512), into L2
                    const float* pfa = (lane < 16 ? ipA : ipB) + 2 * hop + (n - hop) + (lane & 15) * 32;
                    if ((lane & 15) * 32 < hop) asm volatile("prefetch.global.L2 [%0];" :: "l"(pfa));
                }
                // ---- FFT() stages with BlockEnd 1, 2, 4, 8: lane-local on 16 consecutive points ----
                {
                    int off = 0;
#pragma unroll
                    for (int be = 1; be < 16; be <<= 1) {
#pragma unroll
                        for (int blk = 0; blk < 16; blk += 2 * be)
#pragma unroll
                            for (int q = 0; q < be; ++q) butterfly2(R[blk + q], I[blk + q], R[blk + q + be], I[blk + q + be], s_tw[off + q], pk);
                        off += be;
                    }
                }
                // transpose: point lane*16 + r -> (lane >> 4)*256 + r*16 + (lane & 15)
#pragma unroll
                for (int r = 0; r < 16; ++r) sW[psi16(lane * 16 + r)] = make_ulonglong2(R[r], I[r]);
                __syncwarp();
#pragma unroll
                for (int r = 0; r < 16; ++r) { const ulonglong2 v = sW[psi16(b8 * 256 + r * 16 + low4)]; R[r] = v.x; I[r] = v.y; }
                __syncwarp();
                // ---- stages with BlockEnd 16, 32, 64, 128: partner register r | m, twiddle n = (r & (m - 1))*16 + low4 ----
#pragma unroll
                for (int m = 1; m < 16; m <<= 1) {
                    const ulonglong2* t = s_tw + (16 * m - 1) + low4;
#pragma unroll
                    for (int r = 0; r < 16; ++r) {
                        if (r & m) continue;
                        butterfly2(R[r], I[r], R[r | m], I[r | m], t[(r & (m - 1)) * 16], pk);
                    }
                }
#pragma unroll
                for (int r = 0; r < 16; ++r) sW[psi16(b8 * 256 + r * 16 + low4)] = make_ulonglong2(R[r], I[r]);
                __syncwarp();
                // ---- last stage (BlockEnd 256) + RealFFT untangling (fft.cpp:256-275) + cartToPol (:507-515), one pass ----
                // item p: butterflies (p, p+256) and (256-p, 512-p) give X[p], X[p+256], X[256-p], X[512-p]: the inputs of
                // untangle pairs (p, 512-p) and (256-p, 256+p). Lane 0's first item is the odd one out: butterflies (128, 384)
                // and (0, 256), pair (128, 384), DC/Nyquist packing of bin 0, bin 256 left as it is (N/4 is never untangled).
                const size_t oA = ((size_t)cA * a.max_frames + f) * half, oB = ((size_t)cBs * a.max_frames + f) * half;
                float mg[4][4];                                  // [item][A bin1, B bin1, A bin3, B bin3] (+ FULL: written out directly)
                // psi16(32*it + lane) = lane + (lane >> 4) + 34*it;  psi16(256 - 32*it - lane) = u + (u >> 4) + 238 - 34*it with u = 32 - lane
                const int ia0 = lane + (lane >> 4), iq0 = (32 - lane) + ((32 - lane) >> 4) + 238;
                float fgmA = 0.f, famA = 0.f, fxA = 0.f, fgmB = 0.f, famB = 0.f, fxB = 0.f;
                const bool feat = FULL && (a.flatness != nullptr || a.centroid != nullptr);
#pragma unroll
                for (int it = 0; it < 4; ++it) {
                    const int p = it * 32 + lane;
                    const bool special = it == 0 && lane == 0;
                    const int pa = special ? 128 : p, pq = special ? 0 : 256 - p;
                    const int ia = (it == 0 && special) ? psi16(128) : ia0 + 34 * it, iq = (it == 0 && special) ? 0 : iq0 - 34 * it;
                    ulonglong2 Aj = sW[ia], Ak = sW[ia + 272], Bj = sW[iq], Bk = sW[iq + 272];
                    butterfly2(Aj.x, Aj.y, Ak.x, Ak.y, s_tw[255 + pa], pk);
                    butterfly2(Bj.x, Bj.y, Bk.x, Bk.y, s_tw[255 + pq], pk);
                    // pair 1: (i, i3) = (pa, special ? 384 : 512 - p); pair 2 (generic items only): (256 - p, 256 + p)
                    u64 R3 = special ? Ak.x : Bk.x, I3 = special ? Ak.y : Bk.y;
                    untangle2<FULL>(Aj.x, Aj.y, R3, I3, s_uw[pa], pk);
                    u64 U2r = Bj.x, U2i = Bj.y, U23r = Ak.x, U23i = Ak.y;
                    // MFCC-only: pair 2 feeds bin 256 - p alone; when no lane of this item row has it below the mel bank's last
                    // bin the pair is skipped (lane 0's bin 0 is patched in below)
                    const bool skip2 = !FULL && 225 - 32 * it >= a.mf.maxbin;
                    if (!skip2) untangle2<FULL>(U2r, U2i, U23r, U23i, s_uw[special ? 1 : pq], pk);
                    if (it == 0) {      // lane 0: bin 0 = (re + im, re - im) of X[0] (fft.cpp:274-275), bin 256 = X[256]
                        const u64 dcr = add2(Bj.x, Bj.y), dci = sub2(Bj.x, Bj.y);
                        U2r = special ? dcr : U2r; U2i = special ? dci : U2i;
                        U23r = special ? Bk.x : U23r; U23i = special ? Bk.y : U23i;
                    }
                    // bins: b1 <- pair 1 i side, b2 <- pair 1 i3 side, b3 <- pair 2 i side, b4 <- pair 2 i3 side
                    const int b1 = pa, b3 = pq;
                    {
                        float pA, pB;
                        upk2(fma2(mul2(Aj.x, Aj.x), pk.one, mul2(Aj.y, Aj.y)), pA, pB);
                        mg[it][0] = sqrtf(pA); mg[it][1] = sqrtf(pB);
                        upk2(fma2(mul2(U2r, U2r), pk.one, mul2(U2i, U2i)), pA, pB);
                        mg[it][2] = sqrtf(pA); mg[it][3] = sqrtf(pB);
                    }
                    if (FULL) {
                        const int b2 = special ? 384 : 512 - p, b4 = special ? 256 : 256 + p;
                        float m2A, m2B, m4A, m4B;
                        {
                            float pA, pB;
                            upk2(fma2(mul2(R3, R3), pk.one, mul2(I3, I3)), pA, pB);
                            m2A = sqrtf(pA); m2B = sqrtf(pB);
                            upk2(fma2(mul2(U23r, U23r), pk.one, mul2(U23i, U23i)), pA, pB);
                            m4A = sqrtf(pA); m4B = sqrtf(pB);
                        }
                        const int bb[4] = {b1, b2, b3, b4};
                        const u64 re[4] = {Aj.x, R3, U2r, U23r}, im[4] = {Aj.y, I3, U2i, U23i};
                        const float mA[4] = {mg[it][0], m2A, mg[it][2], m4A}, mB[4] = {mg[it][1], m2B, mg[it][3], m4B};
#pragma unroll
                        for (int k = 0; k < 4; ++k) {
                            float reA, reB, imA, imB;
                            upk2(re[k], reA, reB); upk2(im[k], imA, imB);
                            const int b = bb[k];
                            if (a.re) { if (liveA) a.re[oA + b] = reA; if (liveB) a.re[oB + b] = reB; }
                            if (a.im) { if (liveA) a.im[oA + b] = imA; if (liveB) a.im[oB + b] = imB; }
                            if (a.mags) { if (liveA) a.mags[oA + b] = mA[k]; if (liveB) a.mags[oB + b] = mB[k]; }
                            if (a.phases) { if (liveA) a.phases[oA + b] = atan2f(imA, reA); if (liveB) a.phases[oB + b] = atan2f(imB, reB); }
                            // fft::convToDB, src/libs/fft.cpp:526-534: float log10 of (mag + 1), scaled in double, stored as float
                            if (a.mags_db) {
                                if (liveA) a.mags_db[oA + b] = (double)mA[k] < 0.000001 ? 0.f : (float)(20.0 * (double)log10f(__fadd_rn(mA[k], 1.f)));
                                if (liveB) a.mags_db[oB + b] = (double)mB[k] < 0.000001 ? 0.f : (float)(20.0 * (double)log10f(__fadd_rn(mB[k], 1.f)));
                            }
                            if (feat) {     // maxiFFT::spectralFlatness / spectralCentroid, src/libs/maxiFFT.cpp:113-132 (lane-strided partial sums)
                                if (mA[k] != 0.f) fgmA = __fadd_rn(fgmA, logf(mA[k]));
                                famA = __fadd_rn(famA, mA[k]); fxA = __fadd_rn(fxA, __fmul_rn(fabsf(mA[k]), (float)b));
                                if (mB[k] != 0.f) fgmB = __fadd_rn(fgmB, logf(mB[k]));
                                famB = __fadd_rn(famB, mB[k]); fxB = __fadd_rn(fxB, __fmul_rn(fabsf(mB[k]), (float)b));
                            }
                        }
                        // the mel stage may read any bin: all four magnitudes go to shared memory below
                        mg[it][0] = mA[0]; mg[it][1] = mB[0]; mg[it][2] = mA[2]; mg[it][3] = mB[2];
                        // (b2 / b4 magnitudes are parked in the untangle outputs' registers)
                        Ak.x = pk2(m2A, m2B); Ak.y = pk2(m4A, m4B);
                        // keep them for the write after the pass
                        R[it] = Ak.x; I[it] = Ak.y;
                    }
                }
                __syncwarp();                                    // every lane has read its points: the area becomes d_mag[2][512]
#pragma unroll
                for (int it = 0; it < 4; ++it) {
                    const int p = it * 32 + lane;
                    const bool special = it == 0 && lane == 0;
                    const int b1 = special ? 128 : p, b3 = special ? 0 : 256 - p;
                    d_mag[b1] = (double)mg[it][0]; d_mag[half + b1] = (double)mg[it][1];
                    d_mag[b3] = (double)mg[it][2]; d_mag[half + b3] = (double)mg[it][3];
                    if (FULL) {
                        const int b2 = special ? 384 : 512 - p, b4 = special ? 256 : 256 + p;
                        float x, y;
                        upk2(R[it], x, y); d_mag[b2] = (double)x; d_mag[half + b2] = (double)y;
                        upk2(I[it], x, y); d_mag[b4] = (double)x; d_mag[half + b4] = (double)y;
                    }
                }
                if (feat) {
#pragma unroll
                    for (int m = 16; m >= 1; m >>= 1) {
                        fgmA = __fadd_rn(fgmA, __shfl_xor_sync(0xffffffffu, fgmA, m)); famA = __fadd_rn(famA, __shfl_xor_sync(0xffffffffu, famA, m));
                        fxA = __fadd_rn(fxA, __shfl_xor_sync(0xffffffffu, fxA, m));
                        fgmB = __fadd_rn(fgmB, __shfl_xor_sync(0xffffffffu, fgmB, m)); famB = __fadd_rn(famB, __shfl_xor_sync(0xffffffffu, famB, m));
                        fxB = __fadd_rn(fxB, __shfl_xor_sync(0xffffffffu, fxB, m));
                    }
                    if (lane == 0) {
                        const size_t ofA = (size_t)cA * a.max_frames + f, ofB = (size_t)cBs * a.max_frames + f;
                        if (a.flatness) {
                            if (liveA) a.flatness[ofA] = (famA / (float)half) != 0.f ? expf(fgmA / (float)half) / (famA / (float)half) : 0.f;
                            if (liveB) a.flatness[ofB] = (famB / (float)half) != 0.f ? expf(fgmB / (float)half) / (famB / (float)half) : 0.f;
                        }
                        if (a.centroid) {
                            if (liveA) a.centroid[ofA] = famA != 0.f ? __fmul_rn(fxA / famA, a.bin_hz) : 0.f;
                            if (liveB) a.centroid[ofB] = famB != 0.f ? __fmul_rn(fxB / famB, a.bin_hz) : 0.f;
                        }
                    }
                }
                __syncwarp();
                if (FULL && (a.oct_nruns > 0 || a.bark_lim != nullptr)) {
                    // ---- maxiFFTOctaveAnalyzer::calculate (maxiFFT.cpp:264-300) and maxiBark (maxiBark.h:63-113) on the magnitudes
                    // still in shared memory. Octave: one lane per run of bins (the reference's running float sum closes a run ON the
                    // first bin of the next averaging band), then one lane per averaging band for the peak-hold logic; the bands'
                    // averages / peaks / hold counters are per-channel state carried from frame to frame in HBM (this warp walks
                    // the channel's frames in order). Bark: one lane per band, double sums in bin order, pow, max, total.
                    double* bsc = (double*)sW + 1040;                         // 24 doubles of scratch behind d_mag[2][512] (+ skew)
#pragma unroll 1
                    for (int fr = 0; fr < 2; ++fr) {
                        const int c = fr ? cB : cA;
                        if (c >= C) break;
                        if (RAGGED && !(fr ? liveB : liveA)) continue;     // past this channel's last frame: its state stays
                        const double* mag = d_mag + fr * half;                // floats stored as doubles: the conversions back are exact
                        const size_t of = (size_t)c * a.max_frames + f;
                        if (a.oct_nruns > 0) {
                            const int nA = a.oct_navg;
                            float* avs = a.oct_avg_state + (size_t)c * nA; float* pks = a.oct_peak_state + (size_t)c * nA; int* hds = a.oct_hold_state + (size_t)c * nA;
                            for (int r = lane; r < a.oct_nruns; r += 32) {
                                const int4 run = ((const int4*)a.oct_runs)[r];          // first bin, last bin, first band, one past the last band
                                float sum = 0.f;
                                for (int b = run.x; b <= run.y; ++b)
                                    sum = __fadd_rn(sum, __fmul_rn((float)mag[b], __fadd_rn(a.oct_icpt, __fmul_rn((float)b, a.oct_slope))));
                                const float av = __fdiv_rn(sum, (float)(run.y - run.x + 1));
                                for (int j = run.z; j < run.w; ++j) avs[j] = av;
                            }
                            __syncwarp();
                            for (int i = lane; i < nA; i += 32) {
                                const float av = avs[i];
                                float pk = pks[i]; int hd = hds[i];
                                if (av >= pk) { pk = av; hd = a.oct_hold; }
                                else { if (hd > 0) hd--; else pk = __fmul_rn(pk, a.oct_decay); }
                                pks[i] = pk; hds[i] = hd;
                                if (a.oct_avg_out) a.oct_avg_out[of * nA + i] = av;
                                if (a.oct_peak_out) a.oct_peak_out[of * nA + i] = pk;
                            }
                            __syncwarp();
                        }
                        if (a.bark_lim != nullptr) {
                            double spec = 0.0;
                            if (lane < 24) {
                                double sum = 0.0;
                                for (int j = a.bark_lim[lane]; j < a.bark_lim[lane + 1]; ++j) sum = __dadd_rn(sum, mag[j]);
                                spec = pow(sum, 0.23);
                                bsc[lane] = spec;
                            }
                            double mx = spec > 0.0 ? spec : 0.0;                   // `if (specific[i] > max) max = specific[i]` from max = 0
#pragma unroll
                            for (int m = 16; m >= 1; m >>= 1) { const double o = __shfl_xor_sync(0xffffffffu, mx, m); mx = o > mx ? o : mx; }
                            __syncwarp();
                            if (lane < 24) {
                                if (a.bark_specific) a.bark_specific[of * 24 + lane] = spec;
                                if (a.bark_relative) a.bark_relative[of * 24 + lane] = spec / mx;
                            }
                            if (lane == 0 && a.bark_total) {
                                double t = 0.0;
                                for (int i = 0; i < 24; ++i) t = __dadd_rn(t, bsc[i]);
                                a.bark_total[of] = t;
                            }
                            __syncwarp();
                        }
                    }
                }
                __syncwarp();
            } else if (a.has_mfcc) {
                for (int k = lane; k < 2 * half; k += 32) d_mag[k] = 0.0;     // a warp without a channel pair contributes silent frames
                __syncwarp();
            }
            if (a.has_mfcc) {
                // ---- maxiMFCC::mfcc (maxiMFCC.h:77-111, maxiMFCC.cpp:48-66) for the 8 frames of this 4-warp group, on the fp64 tensor
                // cores (mma.sync m8n8k4, SASS DMMA). Frame row r of the group = warp r/2, channel A / B = r%2.
                //   mel:  per tile of 8 filters  C[8 x 8] = mags[8 x bins] . W[bins x 8]  over the bins the tile's filters cover
                //         (k-steps of 4 bins; B fragments pre-arranged per (tile, k-step, lane), zero outside the bands), then the
                //         gate and log on the accumulator fragment: melBands = sum > 1e-6 ? log(sum^2) : 0
                //   DCT:  per tile of 8 coefficients  C[8 x 8] = melBands[8 x filters] . D[filters x 8], / numCoeffs
                // The tensor core adds in its own order: results agree with the reference's sequential sums to fp64 reassociation
                // (~1e-15 relative; asserted at 1e-9). Two named barriers per batch and group; the mel rows are double-buffered.
                const int grp = warp >> 2, wg = warp & 3;
                const int row = lane >> 2, kk = lane & 3;
                // Mel tiles of this warp. Whole tiles go round robin from the top (the widest bands first); each costs two logarithms
                // per lane, the expensive part. A last round of one or two tiles is shared by halves -- two warps run the (narrow)
                // tile and each takes the logarithm of one accumulator -- so that 42 filters (six tiles) cost every warp three.
                const int mel_nt = a.mf.mel_ntiles, mel_rem = mel_nt & 3;
                const bool halves = mel_rem == 1 || mel_rem == 2;
                int nt = mel_nt - 1 - wg;                                           // first tile: its descriptor (fragment offset, first bin,
                int4 tile = make_int4(0, 0, 0, 0);                                  // k-steps) is requested before the wait
                if (nt >= 0) tile = __ldg((const int4*)a.mf.mel_tiles + nt);
                group_barrier(1 + grp);                                             // the group's 8 magnitude rows are in shared memory
                double* melbuf = s_mel + (size_t)(bc & 1) * 2 * kStreamWarps * melstride;
                {
                    const double* amag = (const double*)((ulonglong2*)(sm + L.off_work) + (size_t)(4 * grp + (row >> 1)) * (half + half / 16)) +
                                         4 * (row >> 1) + (row & 1) * half + kk;      // row r: warp 4*grp + r/2 (skew 4*(r/2)), frame r%2
                    double* mr = melbuf + (size_t)(8 * grp + row) * melstride;
                    const int whole_lo = halves ? mel_rem : 0;                         // tiles below this index are shared by halves
                    while (nt >= whole_lo) {
                        const int ntn = nt - 4;
                        int4 tilen = tile;
                        if (ntn >= 0) tilen = __ldg((const int4*)a.mf.mel_tiles + ntn);   // the next descriptor travels during this tile
                        double c0, c1;
                        dmma_tile(amag + tile.y, a.mf.melf + (size_t)tile.x * 32 + lane, tile.z, c0, c1);
                        const double l0 = log_pos(__dmul_rn(c0, c0)), l1 = log_pos(__dmul_rn(c1, c1));
                        const int f0 = nt * 8 + 2 * kk;
                        if (f0 < nf) mr[f0] = c0 > 0.000001 ? l0 : 0.0;                // melBands = sum > 1e-6 ? log(sum^2) : 0 (maxiMFCC.cpp:64)
                        if (f0 + 1 < nf) mr[f0 + 1] = c1 > 0.000001 ? l1 : 0.0;
                        nt = ntn; tile = tilen;
                    }
                    if (halves) {
                        // rem 2: tile 1 -> warps 0, 1; tile 0 -> warps 2, 3.  rem 1: tile 0 -> warps 0, 1
                        const int ht = mel_rem == 2 ? 1 - (wg >> 1) : (wg < 2 ? 0 : -1);
                        if (ht >= 0) {
                            const int4 th = __ldg((const int4*)a.mf.mel_tiles + ht);
                            double c0, c1;
                            dmma_tile(amag + th.y, a.mf.melf + (size_t)th.x * 32 + lane, th.z, c0, c1);
                            const double c = (wg & 1) ? c1 : c0;
                            const double l = log_pos(__dmul_rn(c, c));
                            const int fi = ht * 8 + 2 * kk + (wg & 1);
                            if (fi < nf) mr[fi] = c > 0.000001 ? l : 0.0;
                        }
                    }
                }
                group_barrier(1 + kStreamWarps / 4 + grp);                          // the group's 8 mel rows are complete, its magnitudes consumed
                const double* arow = melbuf + (size_t)(8 * grp + row) * melstride + kk;
                const int ntiles = (a.mf.coeffs + 7) >> 3, ksteps = L.dct_ksteps;
                const double ncinv = 1.0 / (double)(unsigned)a.mf.coeffs;          // dct(): `/ numCoeffs` (maxiMFCC.h:108-110) as one multiply, <= 1 ulp apart
                for (int nt = 3 - wg; nt < ntiles; nt += 4) {                       // warps 3, 2 first: they had the narrowest mel tiles
                    double c0, c1;
                    dmma_tile(arow, a.mf.dctf + (size_t)nt * ksteps * 32 + lane, ksteps, c0, c1);   // columns >= filters are zero
                    const int fi = 8 * grp + row;                // frame of the CTA's batch: warp fi >> 1, channel A / B = fi & 1
                    const int ch = 2 * (pb * kStreamWarps + (fi >> 1)) + (fi & 1);
                    if (ch < C && (!RAGGED || f < ragged_frames(rg, ch))) {
                        double* o = a.coeffs + ((size_t)ch * a.max_frames + f) * a.mf.coeffs;
                        const int cc = nt * 8 + 2 * kk;
                        if (cc < a.mf.coeffs) o[cc] = __dmul_rn(c0, ncinv);
                        if (cc + 1 < a.mf.coeffs) o[cc + 1] = __dmul_rn(c1, ncinv);
                    }
                }
            }
        }
        // ---- the channels' next assembly buffers: the unconsumed tail of (buffer ++ new samples), maxiFFT.cpp:85-87 applied
        // `frames` times. It goes to the OTHER buffer (double-buffered across calls). ----
        // (RAGGED: per channel, and channels without a frame in this call are left to stft_shift_ragged_kernel)
        if (vA && (RAGGED || (a.newpos > 0 && !tail_done))) {
            const long long consumed = (long long)frames * hop;
#pragma unroll 1
            for (int k = 0; k < 2; ++k) {
                const int c = k ? cB : cA;
                if (c >= C) break;
                const long long rconsumed = (long long)(k ? frB : frA) * hop;
                const int rpos0 = k ? posB : posA, rnewpos = RAGGED ? __ldg(rg.newpos + c) : 0;
                if (RAGGED && (rconsumed == 0 || rnewpos == 0)) continue;
                const float* hsrc = a.hist + (size_t)c * n;
                const float* isrc = a.in + (long long)c * a.stride_c;
                float* nx = a.next + (size_t)c * n;
                const long long fromin = (RAGGED ? rconsumed : consumed) - (RAGGED ? rpos0 : a.pos0);   // first new-sample index of the tail when none of it is history
                if (planar && fromin >= 0 && ((RAGGED ? rnewpos : a.newpos) & 3) == 0 && ((((uintptr_t)(isrc + fromin)) | ((uintptr_t)nx)) & 15) == 0) {
                    for (int i = 4 * lane; i < (RAGGED ? rnewpos : a.newpos); i += 128) __stcs((float4*)(nx + i), ld_stream_f4(isrc + fromin + i));
                } else {
                    for (int i = lane; i < (RAGGED ? rnewpos : a.newpos); i += 32) {
                        const long long s = (RAGGED ? rconsumed : consumed) + i;
                        nx[i] = s < (RAGGED ? rpos0 : a.pos0) ? hsrc[s] : isrc[(s - (RAGGED ? rpos0 : a.pos0)) * a.stride_t];
                    }
                }
            }
        }
    }
}

template <bool FULL>
__global__ void __launch_bounds__(kStreamWarps * 32, kStreamCtasPerSm) stft_stream_ragged_kernel(const StreamArgs sa, const RaggedDev rg) {
    stft_stream_body<FULL, true>(sa, rg);
}

}  // namespace
