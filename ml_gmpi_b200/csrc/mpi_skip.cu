// Opt-in empty-space skipping of the staged forward (gmpi_mpi_build_occupancy, gmpi_mpi_render_fwd_skip_ex): the occupancy-map
// builds and the fp32 and fp16 staged forward kernels with kKeySkip, launched by mpi_render.cu (skip_unit, mpi_kernel_keys.cuh).  A
// translation unit of its own, so that the kernels of mpi_render.cu keep their machine code.  DESIGN.md section 4.1 has the exactness argument.
#include <cuda_runtime.h>
#include <cuda_fp16.h>
#include <stdint.h>

#include <iterator>

#include "../../include/gmpi_mpi_render.h"
#include "mpi_common.cuh"
#include "mpi_fwd_staged.cuh"
#include "mpi_kernel_keys.cuh"

namespace gmpi {

// A texel is occupied when its alpha is any bit pattern but +0 (-0.0 and NaN count as occupied) or a colour value is not finite
// (ElemTraits<E>::nonfinite, on the element's bit pattern U).

// Expanded MPI [P = M*N][4][Ht][Wt]: grid (words, block rows, planes in steps of gridDim.z).  flags != NULL: also the range-check bits
// gmpi_mpi_check_range(_f16) sets, from the same loads and with its test (ElemTraits<E>::out_of_unit).
template <class E, class U = typename ElemTraits<E>::Bits>
__device__ __forceinline__ void occ_expanded(const U* __restrict__ rgba, uint32_t* __restrict__ occ, uint32_t* flags, int P, int Ht,
                                             int Wt, int words, int rows) {
    using T = ElemTraits<E>;
    __shared__ uint32_t s_w[kOccThreads / 32];
    const size_t tex = (size_t)Ht * Wt;
    const int x = blockIdx.x * kOccThreads + threadIdx.x, y0 = blockIdx.y * kOccB;
    uint32_t flag = 0;
    for (int pl = blockIdx.z; pl < P; pl += gridDim.z) {
        bool occupied = false;
        if (x < Wt) {
            const U* base = rgba + (size_t)pl * 4 * tex + x;
            for (int y = y0; y < y0 + kOccB && y < Ht; ++y) {
                const size_t o = (size_t)y * Wt;
                const uint32_t c0 = __ldcs(base + o), c1 = __ldcs(base + tex + o), c2 = __ldcs(base + 2 * tex + o), a = __ldcs(base + 3 * tex + o);
                occupied = occupied || a != 0u || T::nonfinite(c0) || T::nonfinite(c1) || T::nonfinite(c2);
                if (T::out_of_unit(c0) || T::out_of_unit(c1) || T::out_of_unit(c2)) flag |= GMPI_FLAG_RGBA_RANGE;
                if (T::out_of_unit(a)) flag |= GMPI_FLAG_RGBA_RANGE | GMPI_FLAG_ALPHA_RANGE;
            }
        }
        store_occ_word(occupied, occ + ((size_t)pl * rows + blockIdx.y) * words + blockIdx.x, s_w);
    }
    if (flags) {
        flag = __reduce_or_sync(0xffffffffu, flag);
        if (flag && (threadIdx.x & 31) == 0) atomicOr(flags, flag);
    }
}

// Factored MPI: colour rgb [M][3][Ht][Wt] shared by the planes (bg [M][3][Ht][Wt]: the last plane's own, nullable), alpha
// [M][N][Ht][Wt].  Grid (words, block rows, MPIs in steps of gridDim.z).  The colour's finiteness is read once per MPI (an 8-bit row
// mask per thread) and applied to every plane; per plane only alpha is read.
template <class E, class U = typename ElemTraits<E>::Bits>
__device__ __forceinline__ void occ_factored(const U* __restrict__ rgb, const U* __restrict__ bg, const U* __restrict__ alpha,
                                             uint32_t* __restrict__ occ, int M, int N, int Ht, int Wt, int words, int rows) {
    using T = ElemTraits<E>;
    __shared__ uint32_t s_w[kOccThreads / 32];
    const size_t tex = (size_t)Ht * Wt;
    const int x = blockIdx.x * kOccThreads + threadIdx.x, y0 = blockIdx.y * kOccB;
    for (int m = blockIdx.z; m < M; m += gridDim.z) {
        uint32_t nf_rgb = 0, nf_bg = 0;     // bit r: a colour value of texel row y0 + r is not finite
        if (x < Wt) {
            for (int r = 0; r < kOccB && y0 + r < Ht; ++r) {
                const size_t o = (size_t)m * 3 * tex + (size_t)(y0 + r) * Wt + x;
                if (T::nonfinite(__ldg(rgb + o)) || T::nonfinite(__ldg(rgb + o + tex)) || T::nonfinite(__ldg(rgb + o + 2 * tex)))
                    nf_rgb |= 1u << r;
                if (bg && (T::nonfinite(__ldg(bg + o)) || T::nonfinite(__ldg(bg + o + tex)) || T::nonfinite(__ldg(bg + o + 2 * tex))))
                    nf_bg |= 1u << r;
            }
        }
        for (int i = 0; i < N; ++i) {
            bool occupied = false;
            if (x < Wt) {
                occupied = ((bg && i == N - 1) ? nf_bg : nf_rgb) != 0u;
                const U* a = alpha + ((size_t)m * N + i) * tex + x;
                for (int y = y0; y < y0 + kOccB && y < Ht; ++y) occupied = occupied || __ldcs(a + (size_t)y * Wt) != 0u;
            }
            store_occ_word(occupied, occ + (((size_t)m * N + i) * rows + blockIdx.y) * words + blockIdx.x, s_w);
        }
    }
}

}  // namespace gmpi

using namespace gmpi;

extern "C" {

__global__ void __launch_bounds__(kOccThreads)
gmpi_occ_expanded_f32(const uint32_t* rgba, uint32_t* occ, uint32_t* flags, int P, int Ht, int Wt, int words, int rows) {
    occ_expanded<float>(rgba, occ, flags, P, Ht, Wt, words, rows);
}
__global__ void __launch_bounds__(kOccThreads)
gmpi_occ_expanded_f16(const uint16_t* rgba, uint32_t* occ, uint32_t* flags, int P, int Ht, int Wt, int words, int rows) {
    occ_expanded<__half>(rgba, occ, flags, P, Ht, Wt, words, rows);
}
__global__ void __launch_bounds__(kOccThreads)
gmpi_occ_factored_f32(const uint32_t* rgb, const uint32_t* bg, const uint32_t* alpha, uint32_t* occ, int M, int N, int Ht, int Wt,
                      int words, int rows) {
    occ_factored<float>(rgb, bg, alpha, occ, M, N, Ht, Wt, words, rows);
}
__global__ void __launch_bounds__(kOccThreads)
gmpi_occ_factored_f16(const uint16_t* rgb, const uint16_t* bg, const uint16_t* alpha, uint32_t* occ, int M, int N, int Ht, int Wt,
                      int words, int rows) {
    occ_factored<__half>(rgb, bg, alpha, occ, M, N, Ht, Wt, words, rows);
}

// stages the last skipping launch armed empty (gmpi_debug_fwd_skip_stats, through OccMap::skipped)
__device__ unsigned long long gmpi_skip_empty_stages;

}  // extern "C"

// The render kernels of this file, in the order they were first defined here (the order of instantiation can change machine code).
static const RenderKernel kSkipKernels[] = {
    {kKeySkip | kKeyStaged, mpi_fwd_skip_kernel<kKeySkip | kKeyStaged>},
    {kKeySkip | kKeyStaged | kKeyES, mpi_fwd_skip_kernel<kKeySkip | kKeyStaged | kKeyES>},
    {kKeySkip | kKeyStaged | kKeyFac, mpi_fwd_skip_kernel<kKeySkip | kKeyStaged | kKeyFac>},
    {kKeySkip | kKeyStaged | kKeyFac | kKeyES, mpi_fwd_skip_kernel<kKeySkip | kKeyStaged | kKeyFac | kKeyES>},
    {kKeySkip | kKeyStaged | kKeyAC, mpi_fwd_skip_kernel<kKeySkip | kKeyStaged | kKeyAC>},
    {kKeySkip | kKeyStaged | kKeyAC | kKeyES, mpi_fwd_skip_kernel<kKeySkip | kKeyStaged | kKeyAC | kKeyES>},
    {kKeySkip | kKeyStaged | kKeyAC | kKeyFac, mpi_fwd_skip_kernel<kKeySkip | kKeyStaged | kKeyAC | kKeyFac>},
    {kKeySkip | kKeyStaged | kKeyAC | kKeyFac | kKeyES, mpi_fwd_skip_kernel<kKeySkip | kKeyStaged | kKeyAC | kKeyFac | kKeyES>},
    {kKeySkip | kKeyStaged | kKeyF16, mpi_fwd_skip_kernel<kKeySkip | kKeyStaged | kKeyF16>},
    {kKeySkip | kKeyStaged | kKeyF16 | kKeyES, mpi_fwd_skip_kernel<kKeySkip | kKeyStaged | kKeyF16 | kKeyES>},
    {kKeySkip | kKeyStaged | kKeyF16 | kKeyFac, mpi_fwd_skip_kernel<kKeySkip | kKeyStaged | kKeyF16 | kKeyFac>},
    {kKeySkip | kKeyStaged | kKeyF16 | kKeyFac | kKeyES, mpi_fwd_skip_kernel<kKeySkip | kKeyStaged | kKeyF16 | kKeyFac | kKeyES>},
    {kKeySkip | kKeyStaged | kKeyF16 | kKeyAC, mpi_fwd_skip_kernel<kKeySkip | kKeyStaged | kKeyF16 | kKeyAC>},
    {kKeySkip | kKeyStaged | kKeyF16 | kKeyAC | kKeyES, mpi_fwd_skip_kernel<kKeySkip | kKeyStaged | kKeyF16 | kKeyAC | kKeyES>},
    {kKeySkip | kKeyStaged | kKeyF16 | kKeyAC | kKeyFac, mpi_fwd_skip_kernel<kKeySkip | kKeyStaged | kKeyF16 | kKeyAC | kKeyFac>},
    {kKeySkip | kKeyStaged | kKeyF16 | kKeyAC | kKeyFac | kKeyES, mpi_fwd_skip_kernel<kKeySkip | kKeyStaged | kKeyF16 | kKeyAC | kKeyFac | kKeyES>},
};

static cudaError_t skip_stage_counters(unsigned long long** early_stop, unsigned long long** empty) {
    const cudaError_t e = cudaGetSymbolAddress(reinterpret_cast<void**>(early_stop), g_early_stop_skipped);
    return e != cudaSuccess ? e : cudaGetSymbolAddress(reinterpret_cast<void**>(empty), gmpi_skip_empty_stages);
}

const KernelUnit gmpi::skip_unit = {std::begin(kSkipKernels), std::end(kSkipKernels), skip_stage_counters};
