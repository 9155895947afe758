// The mix bus of a voice bank or a voice patch (K3 + K6): one fixed-order reduction of the per-warp mix partials, with
// the exchange of the bus between the GPUs of one box over peer memory (NVLink / NVSwitch) fused in when an mxb_exchange
// is attached -- the path's only inter-GPU step (16 KiB per block and rank). The exchange's buffers and protocol are
// private to exchange.cu. Every function accepts ex == NULL (no exchange) and starts its error messages with `who`.
#pragma once

#include "common.cuh"

namespace mxb {

// mxb_{bank,patch}_set_exchange: the exchange must live on the caller's device
int mix_bus_attach(const mxb_exchange* ex, int device, const char* who);
// before any kernel of a block runs: the exchange is connected to its peers and holds the block's 2 * n_frames bus values
int mix_bus_admit(const mxb_exchange* ex, int n_frames, const char* who);
// mix[t][c] = sum over w of partials[t][c][w] (W warps, n_frames frames) on `s`, summed over the ranks in rank order when
// an exchange is attached; the same bits every run
int mix_bus_reduce(mxb_exchange* ex, const double* partials, int W, int n_frames, double* mix, cudaStream_t s);
// once `s` has been synchronised: MXB_ERR_STATE if a peer's part of a bus did not arrive within the exchange's time-out
int mix_bus_status(mxb_exchange* ex, const char* who);

}  // namespace mxb
