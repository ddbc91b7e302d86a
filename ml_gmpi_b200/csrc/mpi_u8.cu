// 8-bit RGBA MPIs (GMPI_MPI_U8, forward only): the staged forward with and without empty-space skipping, the direct forward and the
// occupancy-map build on an expanded uint8 rgba [M,N,4,Ht,Wt] whose code b stands for b / 255 (to_f32(uint8_t), exact), launched
// by mpi_render.cu (u8_unit, mpi_kernel_keys.cuh).  A translation unit of its own, so that the kernels of mpi_render.cu and
// mpi_skip.cu keep their machine code.
#include <cuda_runtime.h>
#include <cuda_fp16.h>
#include <stdint.h>

#include <iterator>

#include "../../include/gmpi_mpi_render.h"
#include "mpi_common.cuh"
#include "mpi_fwd_staged.cuh"
#include "mpi_fwd_direct.cuh"
#include "mpi_kernel_keys.cuh"

using namespace gmpi;

// The render kernels of this file, in the order they were first defined here (the order of instantiation can change machine code).
static const RenderKernel kU8Kernels[] = {
    {kKeyU8 | kKeyStaged, mpi_fwd_staged_kernel<kKeyU8 | kKeyStaged>},
    {kKeyU8 | kKeySkip | kKeyStaged, mpi_fwd_skip_kernel<kKeyU8 | kKeySkip | kKeyStaged>},
    {kKeyU8, mpi_fwd_direct_kernel<kKeyU8>},
    {kKeyU8 | kKeyStaged | kKeyES, mpi_fwd_staged_kernel<kKeyU8 | kKeyStaged | kKeyES>},
    {kKeyU8 | kKeySkip | kKeyStaged | kKeyES, mpi_fwd_skip_kernel<kKeyU8 | kKeySkip | kKeyStaged | kKeyES>},
    {kKeyU8 | kKeyES, mpi_fwd_direct_kernel<kKeyU8 | kKeyES>},
    {kKeyU8 | kKeyStaged | kKeyAC, mpi_fwd_staged_kernel<kKeyU8 | kKeyStaged | kKeyAC>},
    {kKeyU8 | kKeySkip | kKeyStaged | kKeyAC, mpi_fwd_skip_kernel<kKeyU8 | kKeySkip | kKeyStaged | kKeyAC>},
    {kKeyU8 | kKeyAC, mpi_fwd_direct_kernel<kKeyU8 | kKeyAC>},
    {kKeyU8 | kKeyStaged | kKeyAC | kKeyES, mpi_fwd_staged_kernel<kKeyU8 | kKeyStaged | kKeyAC | kKeyES>},
    {kKeyU8 | kKeySkip | kKeyStaged | kKeyAC | kKeyES, mpi_fwd_skip_kernel<kKeyU8 | kKeySkip | kKeyStaged | kKeyAC | kKeyES>},
    {kKeyU8 | kKeyAC | kKeyES, mpi_fwd_direct_kernel<kKeyU8 | kKeyAC | kKeyES>},
};

extern "C" {

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

static cudaError_t u8_stage_counters(unsigned long long** early_stop, unsigned long long** empty) {
    const cudaError_t e = cudaGetSymbolAddress(reinterpret_cast<void**>(early_stop), g_early_stop_skipped);
    return e != cudaSuccess ? e : cudaGetSymbolAddress(reinterpret_cast<void**>(empty), gmpi_skip_empty_stages);
}

const KernelUnit gmpi::u8_unit = {std::begin(kU8Kernels), std::end(kU8Kernels), u8_stage_counters};
