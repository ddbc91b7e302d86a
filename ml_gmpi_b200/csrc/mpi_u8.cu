// 8-bit RGBA MPIs (GMPI_MPI_U8, forward only): the staged forward with and without empty-space skipping, the direct forward and the
// occupancy-map build on an expanded uint8 rgba [M,N,4,Ht,Wt] whose code b stands for b / 255 (to_f32(uint8_t), exact), launched
// by mpi_render.cu (mpi_fwd_units.cuh declares them).  A translation unit of its own, so that the kernels of mpi_render.cu and
// mpi_skip.cu keep their machine code.
#include <cuda_runtime.h>
#include <cuda_fp16.h>
#include <stdint.h>

#include "../../include/gmpi_mpi_render.h"
#include "mpi_common.cuh"
#include "mpi_fwd_staged.cuh"
#include "mpi_fwd_direct.cuh"
#include "mpi_fwd_units.cuh"

namespace gmpi {

template <bool kAlignCorners, bool kES, bool kSkip>
__device__ __forceinline__ void fwd_staged_u8(const RenderParams& p, const TmaMaps& maps, int tiles_x, int ring_stages, const OccMap& occ) {
    __shared__ uint32_t s_stop[kStopSlots];
    fwd_staged_body<kAlignCorners, false, false, kES, uint8_t, kSkip>(p, maps, tiles_x, ring_stages, kES ? s_stop : nullptr, occ);
}

}  // namespace gmpi

using namespace gmpi;

extern "C" {

// The staged forward: gmpi_fwd_u8_a{align_corners}_e{early stop}, and with empty-space skipping gmpi_fwd_u8_skip_a{..}_e{..}.
#define GMPI_FWD_U8(AC, ES)                                                                                                        \
    __global__ void __launch_bounds__(kStagedThreads, 1)                                                                           \
    gmpi_fwd_u8_a##AC##_e##ES(const RenderParams p, const __grid_constant__ TmaMaps maps, const int tiles_x, const int tiles_y,     \
                              const int ring_stages) {                                                                             \
        fwd_staged_u8<AC, ES, false>(p, maps, tiles_x, ring_stages, OccMap{});                                                     \
    }                                                                                                                              \
    __global__ void __launch_bounds__(kStagedThreads, 1)                                                                           \
    gmpi_fwd_u8_skip_a##AC##_e##ES(const RenderParams p, const __grid_constant__ TmaMaps maps, const int tiles_x,                  \
                                   const int tiles_y, const int ring_stages, const OccMap occ) {                                   \
        fwd_staged_u8<AC, ES, true>(p, maps, tiles_x, ring_stages, occ);                                                           \
    }                                                                                                                              \
    __global__ void __launch_bounds__(kFwdTileW* kFwdTileH) gmpi_fwd_direct_u8_a##AC##_e##ES(const RenderParams p) {               \
        fwd_direct_body<AC, ES, uint8_t>(p);                                                                                       \
    }
GMPI_FWD_U8(0, 0)
GMPI_FWD_U8(0, 1)
GMPI_FWD_U8(1, 0)
GMPI_FWD_U8(1, 1)

// Occupancy map of an expanded uint8 MPI [P = M*N][4][Ht][Wt]: grid (words, block rows, planes in steps of gridDim.z).  Every code is
// finite and inside [0, 1], so a texel is empty iff its alpha byte is 0 (0 / 255 is +0): only the alpha slab is read, and there are no
// range flags to set.  The map equals the map of the fp32 conversion.
__global__ void __launch_bounds__(kOccThreads)
gmpi_occ_expanded_u8(const uint8_t* rgba, uint32_t* occ, int P, int Ht, int Wt, int words, int rows) {
    __shared__ uint32_t s_w[kOccThreads / 32];
    const size_t tex = (size_t)Ht * Wt;
    const int x = blockIdx.x * kOccThreads + threadIdx.x, y0 = blockIdx.y * kOccB;
    for (int pl = blockIdx.z; pl < P; pl += gridDim.z) {
        bool occupied = false;
        if (x < Wt) {
            const uint8_t* a = rgba + ((size_t)pl * 4 + 3) * tex + x;
            for (int y = y0; y < y0 + kOccB && y < Ht; ++y) occupied = occupied || __ldcs(a + (size_t)y * Wt) != 0;
        }
        store_occ_word(occupied, occ + ((size_t)pl * rows + blockIdx.y) * words + blockIdx.x, s_w);
    }
}

// Test hook (gmpi_debug_u8_codes): out[b] = to_f32(b) for the 256 codes, the device build of the conversion.
__global__ void gmpi_u8_codes(float* out) { out[threadIdx.x] = to_f32((uint8_t)threadIdx.x); }

// stages the last skipping launch of this file's kernels armed empty (gmpi_debug_fwd_skip_stats, through OccMap::skipped)
__device__ unsigned long long gmpi_skip_empty_stages;

}  // extern "C"

cudaError_t gmpi::u8_stage_counters(unsigned long long** early_stop, unsigned long long** empty) {
    const cudaError_t e = cudaGetSymbolAddress(reinterpret_cast<void**>(early_stop), g_early_stop_skipped);
    return e != cudaSuccess ? e : cudaGetSymbolAddress(reinterpret_cast<void**>(empty), gmpi_skip_empty_stages);
}
