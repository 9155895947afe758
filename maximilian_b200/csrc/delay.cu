// K2 dispatcher: picks the instantiation (delay_k_*.cu) for a bank with a maxiDelayline stage.
#include "delay_kernels.cuh"

namespace mxb {

int delay_bank_warps(int V) { return (V + 31) / 32; }   // warps that own at least one voice

int launch_delay_bank(const BankArgs& a, const DelayArgs& d, int filt_kind, bool svf_lp, int env, bool out, bool mix, cudaStream_t s) {
    const int saw = a.osc_kind == MXB_OSC_SAW;
    const int outmode = !out ? 0 : (a.out_f32 ? 2 : 1);      // DL_OUT_NONE / F64 / F32
    if (a.freq_tv || a.cutoff_tv) {      // per-sample frequency / cutoff: the modulated instantiations
        switch (filt_kind) {
            case MXB_FILT_NONE:   return launch_delay_none_mod(a, d, saw, env, outmode, mix, s);
            case MXB_FILT_LORES:  return launch_delay_lores_mod(a, d, saw, env, outmode, mix, s);
            case MXB_FILT_HIRES:  return launch_delay_hires_mod(a, d, saw, env, outmode, mix, s);
            case MXB_FILT_SVF:    return svf_lp ? launch_delay_svf_lp_mod(a, d, saw, env, outmode, mix, s)
                                                : launch_delay_svf_mod(a, d, saw, env, outmode, mix, s);
            case MXB_FILT_BIQUAD: return launch_delay_biquad_mod(a, d, saw, env, outmode, mix, s);
            default: break;
        }
    } else {
        switch (filt_kind) {
            case MXB_FILT_NONE:   return launch_delay_none(a, d, saw, env, outmode, mix, s);
            case MXB_FILT_LORES:  return launch_delay_lores(a, d, saw, env, outmode, mix, s);
            case MXB_FILT_HIRES:  return launch_delay_hires(a, d, saw, env, outmode, mix, s);
            case MXB_FILT_SVF:    return svf_lp ? launch_delay_svf_lp(a, d, saw, env, outmode, mix, s)
                                                : launch_delay_svf(a, d, saw, env, outmode, mix, s);
            case MXB_FILT_BIQUAD: return launch_delay_biquad(a, d, saw, env, outmode, mix, s);
            default: break;
        }
    }
    set_error("launch_delay_bank: filt_kind %d", filt_kind);
    return MXB_ERR_UNSUPPORTED;
}

}  // namespace mxb
