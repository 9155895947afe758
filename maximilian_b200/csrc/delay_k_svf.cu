// Explicit instantiations of the K2 delay-line bank kernel for FILT_T_SVF (see delay_impl.cuh).
#include "delay_impl.cuh"

namespace mxb {
int launch_delay_svf(const BankArgs& a, const DelayArgs& d, int osc_saw, int env, int outmode, bool mix, cudaStream_t s) {
    return launch_delay_filt<FILT_T_SVF>(a, d, osc_saw, env, outmode, mix, s);
}
}  // namespace mxb
