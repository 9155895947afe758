// The K2 delay-line bank kernel's instantiations for one filter family and MODK: build.py compiles this file once per family and
// MODK, with -DMXB_FILT=FILT_T_* -DMXB_MODK=0|1, into delay_k_<family>.o / delay_km_<family>.o, so that they compile in parallel
// (and the block-constant kernels are compiled apart from the modulated ones). See delay_impl.cuh.
#include "delay_impl.cuh"

#if !defined(MXB_FILT) || !defined(MXB_MODK)
#error "delay_k.cu is compiled once per filter family and MODK with -DMXB_FILT=FILT_T_* -DMXB_MODK=0|1"
#endif

namespace mxb {

// outmode: DL_OUT_*; at least one of outmode / mix is set
template <int FILT, bool MODK>
int launch_delay_filt(const BankArgs& a, const DelayArgs& d, int osc_saw, int env, int outmode, bool mix, cudaStream_t s) {
#define MXB_D3(O, E)                                                                                 \
    do {                                                                                             \
        if (outmode == DL_OUT_F64)      return mix ? launch_delay_one<O, FILT, E, DL_OUT_F64, true, MODK>(a, d, s)   \
                                                   : launch_delay_one<O, FILT, E, DL_OUT_F64, false, MODK>(a, d, s); \
        else if (outmode == DL_OUT_F32) return mix ? launch_delay_one<O, FILT, E, DL_OUT_F32, true, MODK>(a, d, s)   \
                                                   : launch_delay_one<O, FILT, E, DL_OUT_F32, false, MODK>(a, d, s); \
        else                            return launch_delay_one<O, FILT, E, DL_OUT_NONE, true, MODK>(a, d, s);       \
    } while (0)
    if (osc_saw) { if (env) MXB_D3(OSC_T_SAW, 1); else MXB_D3(OSC_T_SAW, 0); }
    else         { if (env) MXB_D3(OSC_T_GENERIC, 1); else MXB_D3(OSC_T_GENERIC, 0); }
#undef MXB_D3
}

template int launch_delay_filt<MXB_FILT, MXB_MODK>(const BankArgs&, const DelayArgs&, int, int, int, bool, cudaStream_t);

}  // namespace mxb
