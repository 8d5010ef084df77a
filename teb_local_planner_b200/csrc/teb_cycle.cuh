/*
 * teb_cycle.cuh — the controller steps around plan() for every band of a batch (tebgpu_backup_modes / _device,
 * tebgpu_finish_cycle / _device). The per-band routines are in teb_cycle.h; the contract is at TebCycleArgs in
 * include/teb_b200.h.
 *
 *   k_backup_modes  one thread per band, CYCLE_THREADS bands per CTA
 *   k_finish_cycle  one thread per band, CYCLE_THREADS bands per CTA
 *
 * One thread per band: the detector's means must be summed in the ring's order to match the reference bit for bit,
 * and both steps are a few dozen operations per band, so a wider mapping would only add shuffles.
 */
#pragma once

#include "teb_cycle.h"

namespace tebgpu {

constexpr int CYCLE_THREADS = 128;

__global__ void __launch_bounds__(CYCLE_THREADS) k_backup_modes(const TebCycleArgs a, const TebCycleLimits L, int B) {
  const int b = blockIdx.x * CYCLE_THREADS + threadIdx.x;
  if (b < B) teb_cycle_backup_band(a, L, b, B);
}

__global__ void __launch_bounds__(CYCLE_THREADS) k_finish_cycle(const TebCycleArgs a, const TebCycleLimits L, int32_t* n,
                                                                const int32_t* status, const double* chi2, int B) {
  const int b = blockIdx.x * CYCLE_THREADS + threadIdx.x;
  if (b < B) teb_cycle_finish_band(a, L, n, status, chi2, b);
}

}  // namespace tebgpu
