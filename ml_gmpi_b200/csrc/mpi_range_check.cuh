// Range check of an fp32 or fp16 MPI (gmpi_mpi_check_range, gmpi_mpi_check_range_f16): one streaming pass over rgba, testing each
// element's bit pattern (ElemTraits<E>::out_of_unit).  Launched by mpi_render.cu.
#pragma once
#include <string.h>

#include "../../include/gmpi_mpi_render.h"
#include "mpi_fwd_staged.cuh"

namespace gmpi {

// One slab = one (mpi, plane, channel) image of `slab` loads; channel = slab % 4.  L: the load, 16 bytes (uint4) when every slab is a
// whole number of them on an aligned base, else one element (ElemTraits<E>::Bits).  An fp16 load of 16 bytes tests its words as
// (low half, high half) pairs, every other load its elements in turn: the forms the four kernels this template replaced had, which
// keep their machine code.
template <class E, class L>
__global__ void __launch_bounds__(256)
mpi_check_range_kernel(const L* __restrict__ rgba, size_t n_slabs, size_t slab, uint32_t* flags) {
    using T = ElemTraits<E>;
    using Bits = typename T::Bits;
    constexpr int kPerLoad = sizeof(L) / sizeof(Bits);
    uint32_t flag = 0;
    const size_t total = n_slabs * slab;
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
        const L x = __ldcs(rgba + i);
        bool out = false;
        if constexpr (kPerLoad == 8) {
            uint32_t w[4];
            memcpy(w, &x, sizeof(w));
#pragma unroll
            for (int k = 0; k < 4; ++k) out = out || T::out_of_unit(w[k] & 0xffffu) || T::out_of_unit(w[k] >> 16);
        } else {
            Bits b[kPerLoad];
            memcpy(b, &x, sizeof(b));
#pragma unroll
            for (int k = 0; k < kPerLoad; ++k)
                if (T::out_of_unit(b[k])) { out = true; break; }
        }
        if (out) flag |= (((i / slab) & 3) == 3) ? (GMPI_FLAG_ALPHA_RANGE | GMPI_FLAG_RGBA_RANGE) : GMPI_FLAG_RGBA_RANGE;
    }
    if constexpr (kPerLoad > 1) {
        flag = __reduce_or_sync(0xffffffffu, flag);
        if (flag && (threadIdx.x & 31) == 0) atomicOr(flags, flag);
    } else if (flag) {
        atomicOr(flags, flag);
    }
}

}  // namespace gmpi
