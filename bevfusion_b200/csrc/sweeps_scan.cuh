// The per-sample scan of the sweep assemblers' tile counts, shared by lidar_sweeps.cu and radar_sweeps.cu.
// Internal header.
#pragma once
#include "common.cuh"

namespace bevb200 {

// One CTA per sample: tile_counts [batch, len] int32, in (entry, tile) order, become exclusive offsets in place;
// counts[b] = min(total, cap), and BEVB200_SWEEPS_OVERFLOW goes into *status when a sample's total exceeds cap.
int sweeps_scan(int32_t *tile_counts, int batch, int len, int cap, int32_t *counts, int32_t *status,
                cudaStream_t st);

}  // namespace bevb200
