// What mpi_skip.cu (empty-space skipping) and mpi_u8.cu (uint8 MPIs, GMPI_MPI_U8) define for mpi_render.cu, which launches their
// kernels.  The three files are separate translation units of the one library: without -rdc ptxas compiles each file's device code
// on its own, so kernels added to one file cannot change the machine code of another's.  Both files include this header, so a
// definition that does not match its declaration here does not compile.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "mpi_fwd_staged.cuh"

namespace gmpi {
// The addresses on the current device of the file's stage counters: its own copy of g_early_stop_skipped (mpi_fwd_staged.cuh),
// which its early-stop kernels count into, and its gmpi_skip_empty_stages, which the library passes to its skipping kernels.
cudaError_t skip_stage_counters(unsigned long long** early_stop, unsigned long long** empty);     // mpi_skip.cu
cudaError_t u8_stage_counters(unsigned long long** early_stop, unsigned long long** empty);       // mpi_u8.cu
}  // namespace gmpi

extern "C" {

#define GMPI_STAGED_ARGS gmpi::RenderParams, const __grid_constant__ gmpi::TmaMaps, int, int, int

// mpi_skip.cu: the occupancy-map builds, and the staged forward with skipping, gmpi_fwd_skip_a{align_corners}_x{factored}_e{early
// stop}_{f32|f16}
__global__ void gmpi_occ_expanded_f32(const uint32_t*, uint32_t*, uint32_t*, int, int, int, int, int);
__global__ void gmpi_occ_expanded_f16(const uint16_t*, uint32_t*, uint32_t*, int, int, int, int, int);
__global__ void gmpi_occ_factored_f32(const uint32_t*, const uint32_t*, const uint32_t*, uint32_t*, int, int, int, int, int, int);
__global__ void gmpi_occ_factored_f16(const uint16_t*, const uint16_t*, const uint16_t*, uint32_t*, int, int, int, int, int, int);
#define GMPI_FWD_SKIP_DECL(AC, FAC, ES, TAG) __global__ void gmpi_fwd_skip_a##AC##_x##FAC##_e##ES##_##TAG(GMPI_STAGED_ARGS, gmpi::OccMap);
#define GMPI_FWD_SKIP_DECL_AC(AC, TAG)                                                                                             \
    GMPI_FWD_SKIP_DECL(AC, 0, 0, TAG) GMPI_FWD_SKIP_DECL(AC, 0, 1, TAG) GMPI_FWD_SKIP_DECL(AC, 1, 0, TAG) GMPI_FWD_SKIP_DECL(AC, 1, 1, TAG)
GMPI_FWD_SKIP_DECL_AC(0, f32)
GMPI_FWD_SKIP_DECL_AC(1, f32)
GMPI_FWD_SKIP_DECL_AC(0, f16)
GMPI_FWD_SKIP_DECL_AC(1, f16)
#undef GMPI_FWD_SKIP_DECL_AC
#undef GMPI_FWD_SKIP_DECL

// mpi_u8.cu: the staged forward gmpi_fwd_u8_a{align_corners}_e{early stop} (with skipping gmpi_fwd_u8_skip_a{..}_e{..}), the direct
// forward gmpi_fwd_direct_u8_a{..}_e{..}, the occupancy-map build and the conversion hook
#define GMPI_FWD_U8_DECL(AC, ES)                                                                                                   \
    __global__ void gmpi_fwd_u8_a##AC##_e##ES(GMPI_STAGED_ARGS);                                                                   \
    __global__ void gmpi_fwd_u8_skip_a##AC##_e##ES(GMPI_STAGED_ARGS, gmpi::OccMap);                                                \
    __global__ void gmpi_fwd_direct_u8_a##AC##_e##ES(gmpi::RenderParams);
GMPI_FWD_U8_DECL(0, 0)
GMPI_FWD_U8_DECL(0, 1)
GMPI_FWD_U8_DECL(1, 0)
GMPI_FWD_U8_DECL(1, 1)
#undef GMPI_FWD_U8_DECL
__global__ void gmpi_occ_expanded_u8(const uint8_t*, uint32_t*, int, int, int, int, int);
__global__ void gmpi_u8_codes(float*);

#undef GMPI_STAGED_ARGS

}  // extern "C"
