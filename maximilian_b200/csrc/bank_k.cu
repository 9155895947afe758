// The K1 bank kernel's instantiations for one filter family: build.py compiles this file once per family, with -DMXB_FILT=FILT_T_*,
// into bank_k_<family>.o, so that the families compile in parallel. See bank_kernels.cuh.
#include "bank_kernels.cuh"

#ifndef MXB_FILT
#error "bank_k.cu is compiled once per filter family with -DMXB_FILT=FILT_T_*"
#endif

namespace mxb {

template <int FILT>
int launch_bank_filt(const BankArgs& a, int osc_t, int env, bool out, bool mix, int grid, size_t smem, cudaStream_t s) {
    // the mix tiles of a 128-thread CTA (33 KB) stay below the 48 KB default of dynamic shared memory: no opt-in needed
    static_assert(sizeof(double) * (kBankBlock / 32) * 2 * kMixTT * 33 <= 48 * 1024, "K1 mix tiles exceed 48 KB");
#define MXB_L3ME(O, E, M)                                                                                 \
    do {                                                                                                  \
        if (out && mix)  bank_kernel<O, FILT, E, true, true, M><<<grid, kBankBlock, smem, s>>>(a);         \
        else if (out)    bank_kernel<O, FILT, E, true, false, M><<<grid, kBankBlock, 0, s>>>(a);           \
        else             bank_kernel<O, FILT, E, false, true, M><<<grid, kBankBlock, smem, s>>>(a);        \
    } while (0)
#define MXB_L3M(O, M) do { if (env) MXB_L3ME(O, 1, M); else MXB_L3ME(O, 0, M); } while (0)
    constexpr bool kCutoffMod = FILT == FILT_T_LORES || FILT == FILT_T_HIRES || FILT == FILT_T_SVF || FILT == FILT_T_SVF_LP;
    if (a.cutoff_tv && !kCutoffMod) { set_error("bank_kernel: per-sample cutoff is not built for this filter"); return MXB_ERR_UNSUPPORTED; }
#define MXB_L2(O)                                                                                         \
    do {                                                                                                  \
        if (a.cutoff_tv) { if constexpr (kCutoffMod) { if (a.freq_tv) MXB_L3M(O, 3); else MXB_L3M(O, 2); } } \
        else if (a.freq_tv) MXB_L3M(O, 1);                                                                \
        else MXB_L3M(O, 0);                                                                               \
    } while (0)
    switch (osc_t) {
        case OSC_T_SINE:   MXB_L2(OSC_T_SINE); break;
        case OSC_T_PHASOR: MXB_L2(OSC_T_PHASOR); break;
        case OSC_T_SAW:    MXB_L2(OSC_T_SAW); break;
        default:           MXB_L2(OSC_T_GENERIC); break;
    }
#undef MXB_L2
#undef MXB_L3M
#undef MXB_L3ME
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) { set_error("bank_kernel launch: %s", cudaGetErrorString(e)); return MXB_ERR_CUDA; }
    return MXB_OK;
}

template int launch_bank_filt<MXB_FILT>(const BankArgs&, int, int, bool, bool, int, size_t, cudaStream_t);

}  // namespace mxb
