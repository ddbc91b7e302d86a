// The render kernels' keys, and what the library's three translation units export to mpi_render.cu, which launches their kernels:
// mpi_render.cu itself, mpi_skip.cu (empty-space skipping) and mpi_u8.cu (uint8 MPIs, GMPI_MPI_U8).  Without -rdc ptxas compiles
// each file's device code on its own, so kernels added to one file cannot change the machine code of another's.
#pragma once
#include <cuda_runtime.h>
#include <cuda_fp16.h>
#include <stdint.h>
#include <type_traits>

namespace gmpi {

// What picks a render kernel: the bits of its variant.  kKeyStaged: a persistent TMA kernel (the staged forward, the box backward).
// The direct forward's key has no kKeyFac and no kKeyEmit, and the direct backward's no kKeyFac: those kernels read both at run time.
// kKeySkip: empty-space skipping (the kernels of mpi_skip.cu, or of mpi_u8.cu with kKeyU8).  kKeyU8: a uint8 MPI (mpi_u8.cu).
enum : uint32_t {
    kKeyAC = 1, kKeyFac = 2, kKeyEmit = 4, kKeyES = 8, kKeyF16 = 16, kKeyStaged = 32, kKeyBwd = 64, kKeyDet = 128, kKeySkip = 256,
    kKeyU8 = 512
};

// A key as the kernel bodies take it: their template arguments, and the MPI's element type.
template <uint32_t K>
struct KeyTraits {
    static constexpr bool kAlignCorners = (K & kKeyAC) != 0, kFactored = (K & kKeyFac) != 0, kEmitT = (K & kKeyEmit) != 0,
                          kES = (K & kKeyES) != 0, kSkip = (K & kKeySkip) != 0, kDet = (K & kKeyDet) != 0;
    using Elem = std::conditional_t<(K & kKeyU8) != 0, uint8_t, std::conditional_t<(K & kKeyF16) != 0, __half, float>>;
};

struct RenderKernel {
    uint32_t key;
    const void* kernel;
    template <class... A>
    RenderKernel(uint32_t k, void (*f)(A...)) : key(k), kernel(reinterpret_cast<const void*>(f)) {}
};

// The render kernels one translation unit defines, each listed once, and the addresses on the current device of the unit's stage
// counters: its own copy of g_early_stop_skipped (mpi_fwd_staged.cuh), which its early-stop kernels count into, and its
// gmpi_skip_empty_stages, which its skipping kernels count into (nullptr in a unit without skipping kernels).
struct KernelUnit {
    const RenderKernel *begin, *end;
    cudaError_t (*stage_counters)(unsigned long long** early_stop, unsigned long long** empty);
};
extern const KernelUnit render_unit;   // mpi_render.cu: fp32 and fp16 without skipping, and the backward
extern const KernelUnit skip_unit;     // mpi_skip.cu: fp32 and fp16 with skipping
extern const KernelUnit u8_unit;       // mpi_u8.cu: every uint8 kernel

}  // namespace gmpi

// The kernels of mpi_skip.cu and mpi_u8.cu that are not render kernels: mpi_render.cu launches them by their own symbols through
// launch_kernel, which checks each launch's arguments against these declarations.  Their files include this header, so a definition
// that does not match its declaration here does not compile.
extern "C" {
// mpi_skip.cu: the occupancy-map builds
__global__ void gmpi_occ_expanded_f32(const uint32_t*, uint32_t*, uint32_t*, int, int, int, int, int);
__global__ void gmpi_occ_expanded_f16(const uint16_t*, uint32_t*, uint32_t*, int, int, int, int, int);
__global__ void gmpi_occ_factored_f32(const uint32_t*, const uint32_t*, const uint32_t*, uint32_t*, int, int, int, int, int, int);
__global__ void gmpi_occ_factored_f16(const uint16_t*, const uint16_t*, const uint16_t*, uint32_t*, int, int, int, int, int, int);
// mpi_u8.cu: the occupancy-map build and the conversion hook
__global__ void gmpi_occ_expanded_u8(const uint8_t*, uint32_t*, int, int, int, int, int);
__global__ void gmpi_u8_codes(float*);
}  // extern "C"
