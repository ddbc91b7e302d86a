// Minimal TMA bring-up matrix (diagnostics): one CTA, one box load, print result.  argv[1] = variant bits:
//  1: descriptor in global memory (else __grid_constant__ param)   2: 2-D map (else 3-D)
//  4: box width 64 (else 72)   8: negative start coordinate   16: 4-D (x, channel, y, plane) map
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include "../ml_gmpi_b200/csrc/tma_utils.cuh"
using namespace gmpi;

__global__ void k(const __grid_constant__ CUtensorMap pmap, const CUtensorMap* gmap, int use_g, int rank, int x0, int bytes, float* out) {
    extern __shared__ __align__(1024) unsigned char smem[];
    __shared__ __align__(8) uint64_t bar;
    float* buf = reinterpret_cast<float*>(smem);
    if (threadIdx.x == 0) { mbar_init(&bar, 1); fence_mbar_init(); }
    __syncthreads();
    if (threadIdx.x == 0) {
        const CUtensorMap* m = use_g ? gmap : &pmap;
        mbar_arrive_expect_tx(&bar, bytes);
        if (rank == 2) {
            asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
                         ::"r"(smem_u32(buf)), "l"(m), "r"(smem_u32(&bar)), "r"(x0), "r"(5) : "memory");
        } else if (rank == 3) {
            tma_load_3d(buf, m, &bar, x0, 5, 1);
        } else {
            tma_load_4d(buf, m, &bar, x0, 0, 5, 1);
        }
    }
    mbar_wait(&bar, 0);
    if (threadIdx.x < 8) out[threadIdx.x] = buf[threadIdx.x];
}

int main(int argc, char** argv) {
    int var = argc > 1 ? atoi(argv[1]) : 0;
    const int Ht = 256, Wt = 256, S = 16;
    size_t n = (size_t)S * Ht * Wt;
    float* h = (float*)malloc(n * 4);
    for (size_t i = 0; i < n; ++i) h[i] = (float)(i % 100003);
    float *d, *out; cudaMalloc(&d, n * 4); cudaMemcpy(d, h, n * 4, cudaMemcpyHostToDevice); cudaMalloc(&out, 64);
    const int bw = (var & 4) ? 64 : 72, rows = 4;
    CUtensorMap map; memset(&map, 0, sizeof(map));
    int rank = (var & 16) ? 4 : ((var & 2) ? 2 : 3), r, bytes;
    if (rank == 4) { r = encode_plane_map(&map, d, MapElem{CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 4}, S / 4, Ht, Wt, bw, rows); bytes = bw * 4 * rows * 4; }
    else if (rank == 3) { r = encode_slab_map(&map, d, MapElem{CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 4}, S, Ht, Wt, bw, rows, 4); bytes = bw * rows * 4 * 4; }
    else {
        EncodeTiledFn fn = get_encode_fn();
        cuuint64_t dims[2] = {(cuuint64_t)Wt, (cuuint64_t)Ht * S}; cuuint64_t strides[1] = {(cuuint64_t)Wt * 4};
        cuuint32_t box[2] = {(cuuint32_t)bw, (cuuint32_t)rows}; cuuint32_t es[2] = {1, 1};
        r = (int)fn(&map, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, d, dims, strides, box, es, CU_TENSOR_MAP_INTERLEAVE_NONE,
                    CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
        bytes = bw * rows * 4;
    }
    printf("variant %d rank %d bw %d encode=%d desc:", var, rank, bw, r);
    for (int i = 0; i < 16; ++i) printf(" %016llx", ((unsigned long long*)&map)[i]);
    printf("\n");
    CUtensorMap* gmap; cudaMalloc(&gmap, sizeof(map)); cudaMemcpy(gmap, &map, sizeof(map), cudaMemcpyHostToDevice);
    const int x0 = (var & 8) ? -3 : 8;
    k<<<1, 32, 32768>>>(map, gmap, var & 1, rank, x0, bytes, out);
    cudaError_t le = cudaGetLastError(); if (le != cudaSuccess) printf("  launch error: %s\n", cudaGetErrorString(le));
    cudaError_t e = cudaDeviceSynchronize();
    float ho[8] = {0}; cudaMemcpy(ho, out, 32, cudaMemcpyDeviceToHost);
    printf("  -> %s; out = %g %g %g %g %g (expect row 5 of slab/plane 1 from x0=%d)\n", cudaGetErrorString(e), ho[0], ho[1], ho[2], ho[3], ho[4], x0);
    return 0;
}
