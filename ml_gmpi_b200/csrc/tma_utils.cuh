// TMA (cp.async.bulk.tensor) + mbarrier helpers for sm_90a, and the host-side tensor-map encoder.
// No CUTLASS: raw PTX.  The driver entry point cuTensorMapEncodeTiled is resolved through the runtime
// (cudaGetDriverEntryPoint), so the library links against libcudart only.
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>

namespace gmpi {

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void fence_mbar_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_arrive_if(uint64_t* bar, bool pred) {     // one predicated instruction
    asm volatile("{\n\t.reg .pred q;\n\tsetp.ne.b32 q, %1, 0;\n\t@q mbarrier.arrive.shared::cta.b64 _, [%0];\n\t}" ::"r"(smem_u32(bar)), "r"((int)pred) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
    uint32_t ok;
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(ok)
        : "r"(smem_u32(bar)), "r"(parity)
        : "memory");
    return ok != 0;
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
    while (!mbar_try_wait(bar, parity)) {
    }
}
// For the helper warps (producer, flushers): a failed try_wait comes back within tens of cycles, and a spinning warp takes issue
// slots from the consumers on its scheduler (18 % of all issued instructions in the first backward profile).  Sleep between polls.
__device__ __forceinline__ void mbar_wait_sleep(uint64_t* bar, uint32_t parity) {
    while (!mbar_try_wait(bar, parity)) __nanosleep(96);
}

// 4-D tiled load, coordinates innermost first; completes on `bar` with the box's byte count.
__device__ __forceinline__ void tma_load_4d(void* smem_dst, const CUtensorMap* map, uint64_t* bar, int c0, int c1, int c2, int c3) {
    asm volatile(
        "cp.async.bulk.tensor.4d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], [%2];"
        ::"r"(smem_u32(smem_dst)), "l"(map), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
        : "memory");
}

// 3-D tiled load: coordinates (x, y, z) innermost first; completes on `bar` with the box's byte count.
__device__ __forceinline__ void tma_load_3d(void* smem_dst, const CUtensorMap* map, uint64_t* bar, int x, int y, int z) {
    asm volatile(
        "cp.async.bulk.tensor.3d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];"
        ::"r"(smem_u32(smem_dst)), "l"(map), "r"(smem_u32(bar)), "r"(x), "r"(y), "r"(z)
        : "memory");
}
__device__ __forceinline__ void tma_prefetch_desc(const CUtensorMap* map) {
    asm volatile("prefetch.tensormap [%0];" ::"l"(map) : "memory");
}

// ---------------------------------------------------------------------------------------------------
// host: tensor map over rgba viewed as [M*N*4 slabs][Ht][Wt], box {bw, bh, bc}
// ---------------------------------------------------------------------------------------------------
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                  const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

inline EncodeTiledFn get_encode_fn() {
    // C++11 magic static: resolved once, thread-safe (the ABI is callable from any host thread)
    static const EncodeTiledFn fn = [] {
        void* p = nullptr;
        cudaDriverEntryPointQueryResult qres;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres) == cudaSuccess &&
            qres == cudaDriverEntryPointSuccess)
            return (EncodeTiledFn)p;
        return (EncodeTiledFn) nullptr;
    }();
    return fn;
}

// Element type of a tensor map: its CUtensorMapDataType and size in bytes (the MPI's: ElemTraits<E>::kMap, mpi_fwd_staged.cuh).
struct MapElem {
    CUtensorMapDataType type;
    cuuint64_t bytes;
};

// Returns 0 on success.  Requires 16-byte row strides (Wt a multiple of 16 / el.bytes) and a 16-byte aligned base.
inline int encode_slab_map(CUtensorMap* out, const void* base, MapElem el, uint64_t n_slabs, int Ht, int Wt, int bw, int bh, int bc) {
    EncodeTiledFn fn = get_encode_fn();
    if (!fn) return -1;
    cuuint64_t dims[3] = {(cuuint64_t)Wt, (cuuint64_t)Ht, (cuuint64_t)n_slabs};
    cuuint64_t strides[2] = {(cuuint64_t)Wt * el.bytes, (cuuint64_t)Wt * Ht * el.bytes};
    cuuint32_t box[3] = {(cuuint32_t)bw, (cuuint32_t)bh, (cuuint32_t)bc};
    cuuint32_t estr[3] = {1, 1, 1};
    CUresult r = fn(out, el.type, 3, (void*)base, dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                    CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    return r == CUDA_SUCCESS ? 0 : (int)r;
}

// Tensor map over rgba [M*N planes][4 ch][Ht][Wt] with the dimensions ordered (x, channel, y, plane) so that a box
// {bw, 4, rows, 1} lands in shared memory as [row][channel][x]: rows stay linear however many row-chunks are issued.
inline int encode_plane_map(CUtensorMap* out, const void* base, MapElem el, uint64_t n_planes, int Ht, int Wt, int bw, int rows) {
    EncodeTiledFn fn = get_encode_fn();
    if (!fn) return -1;
    cuuint64_t dims[4] = {(cuuint64_t)Wt, 4, (cuuint64_t)Ht, (cuuint64_t)n_planes};
    cuuint64_t strides[3] = {(cuuint64_t)Wt * Ht * el.bytes, (cuuint64_t)Wt * el.bytes, (cuuint64_t)Wt * Ht * 4 * el.bytes};
    cuuint32_t box[4] = {(cuuint32_t)bw, 4, (cuuint32_t)rows, 1};
    cuuint32_t estr[4] = {1, 1, 1, 1};
    CUresult r = fn(out, el.type, 4, (void*)base, dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                    CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    return r == CUDA_SUCCESS ? 0 : (int)r;
}

// Tensor map over a shared colour image rgb [M][3 ch][Ht][Wt] (factored MPI) with the dimensions ordered (x, channel, y, mpi):
// a box {bw, 3, rows, 1} lands in shared memory as [row][channel][x].
inline int encode_color_map(CUtensorMap* out, const void* base, MapElem el, uint64_t n_mpi, int Ht, int Wt, int bw, int rows) {
    EncodeTiledFn fn = get_encode_fn();
    if (!fn) return -1;
    cuuint64_t dims[4] = {(cuuint64_t)Wt, 3, (cuuint64_t)Ht, (cuuint64_t)n_mpi};
    cuuint64_t strides[3] = {(cuuint64_t)Wt * Ht * el.bytes, (cuuint64_t)Wt * el.bytes, (cuuint64_t)Wt * Ht * 3 * el.bytes};
    cuuint32_t box[4] = {(cuuint32_t)bw, 3, (cuuint32_t)rows, 1};
    cuuint32_t estr[4] = {1, 1, 1, 1};
    CUresult r = fn(out, el.type, 4, (void*)base, dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                    CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    return r == CUDA_SUCCESS ? 0 : (int)r;
}

}  // namespace gmpi
