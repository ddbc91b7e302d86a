// tools/tma_probe.cu -- microbenchmark: how fast can one producer thread per SM stage plane tiles into shared memory
// with cp.async.bulk.tensor (3-D box {BW, RC, 4 channels}) as a function of rows-per-box RC?  (design input for the
// staged forward kernel; not part of the library).  Build: nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o tma_probe tma_probe.cu
#include <cstdio>
#include <cstdlib>
#include <vector>
#include "../ml_gmpi_b200/csrc/tma_utils.cuh"
using namespace gmpi;

constexpr int kStages = 3;

struct ProbeParams {
    int n_planes, Ht, Wt, tile_w, tile_h, bw, bh, rc, n_tiles_x, n_tiles_y, lds_per_px;
};

__global__ void __launch_bounds__(160, 1) probe_kernel(const __grid_constant__ CUtensorMap map, ProbeParams p, float* sink) {
    extern __shared__ __align__(128) unsigned char smem[];
    __shared__ uint64_t full[kStages], empty[kStages];
    const int stage_floats = p.bw * p.bh * 4;
    float* buf = reinterpret_cast<float*>(smem);
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int n_cons_warps = (blockDim.x >> 5) - 1;
    if (threadIdx.x == 0) {
        for (int s = 0; s < kStages; ++s) { mbar_init(&full[s], 1); mbar_init(&empty[s], n_cons_warps); }
        fence_mbar_init();
    }
    __syncthreads();
    const int n_tiles = p.n_tiles_x * p.n_tiles_y;
    const int n_ops = (p.bh + p.rc - 1) / p.rc;
    if (warp == 0) {
        if (lane == 0) {
            int it = 0;
            for (int t = blockIdx.x; t < n_tiles; t += gridDim.x) {
                const int tx = (t % p.n_tiles_x) * p.tile_w - 4, ty = (t / p.n_tiles_x) * p.tile_h - 2;
                for (int pl = 0; pl < p.n_planes; ++pl, ++it) {
                    const int s = it % kStages, ph = (it / kStages) & 1;
                    mbar_wait(&empty[s], ph ^ 1);
                    mbar_arrive_expect_tx(&full[s], (uint32_t)(n_ops * p.bw * p.rc * 4 * 4));
                    for (int o = 0; o < n_ops; ++o)
                        tma_load_3d(buf + (size_t)s * stage_floats + (size_t)o * p.bw * p.rc * 4, &map, &full[s], tx, ty + o * p.rc, pl * 4);
                }
            }
        }
    } else {
        int it = 0;
        float acc = 0.f;
        for (int t = blockIdx.x; t < n_tiles; t += gridDim.x) {
            for (int pl = 0; pl < p.n_planes; ++pl, ++it) {
                const int s = it % kStages, ph = (it / kStages) & 1;
                mbar_wait(&full[s], ph);
                const float* b = buf + (size_t)s * stage_floats;
                // optional consumer load: lds_per_px words per pixel of the tile, conflict-free rows
                const int npx = p.tile_w * p.tile_h;
                for (int px = (warp - 1) * 32 + lane; px < npx; px += n_cons_warps * 32) {
                    const int x = px % p.tile_w, y = px / p.tile_w;
#pragma unroll 4
                    for (int k = 0; k < p.lds_per_px; ++k) acc += b[((k & 3) * p.bh + y + ((k >> 2) & 1)) * p.bw + x + ((k >> 3) & 1)];
                }
                __syncwarp();
                if (lane == 0) mbar_arrive(&empty[s]);
            }
        }
        if (acc == 123.456f) sink[0] = acc;
    }
}

int main(int argc, char** argv) {
    const int N = 96, Ht = 1024, Wt = 1024;
    float* d; float* sink;
    size_t n = (size_t)N * 4 * Ht * Wt;
    cudaMalloc(&d, n * 4); cudaMemset(d, 0, n * 4); cudaMalloc(&sink, 4);
    cudaDeviceProp prop; cudaGetDeviceProperties(&prop, 0);
    printf("device %s SMs %d\n", prop.name, prop.multiProcessorCount);
    cudaEvent_t e0, e1; cudaEventCreate(&e0); cudaEventCreate(&e1);
    struct Cfg { int tw, th, bw, bh, rc, lds, warps; };
    std::vector<Cfg> cfgs;
    // bw*rc*16 bytes per op must be a multiple of 128 (TMA shared-memory destination alignment): bw = 72 works for any rc
    for (int rc : {1, 2, 4, 9, 18, 36}) cfgs.push_back({64, 32, 72, 36, rc, 0, 4});
    for (int rc : {1, 4, 36}) cfgs.push_back({64, 32, 72, 36, rc, 16, 4});
    cfgs.push_back({64, 32, 72, 36, 4, 16, 16});
    cfgs.push_back({64, 32, 72, 36, 36, 16, 16});
    cfgs.push_back({64, 32, 80, 44, 44, 0, 4});
    cfgs.push_back({32, 16, 40, 18, 18, 0, 4});
    cfgs.push_back({32, 16, 40, 18, 18, 16, 8});
    const int only = argc > 1 ? atoi(argv[1]) : -1;
    if (only >= (int)cfgs.size()) return 3;
    for (size_t ci = 0; ci < cfgs.size(); ++ci) {
        if (only >= 0 && (int)ci != only) continue;
        auto c = cfgs[ci];
        CUtensorMap map;
        int r = encode_slab_map(&map, d, MapElem{CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 4}, (uint64_t)N * 4, Ht, Wt, c.bw, c.rc, 4);
        if (r) { printf("encode failed %d\n", r); continue; }
        ProbeParams p{N, Ht, Wt, c.tw, c.th, c.bw, ((c.bh + c.rc - 1) / c.rc) * c.rc, c.rc, Wt / c.tw, Ht / c.th, c.lds};
        size_t smem = (size_t)kStages * p.bw * p.bh * 4 * 4;
        cudaFuncSetAttribute(probe_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        const int threads = 32 * (1 + c.warps);
        for (int rep = 0; rep < 2; ++rep) probe_kernel<<<prop.multiProcessorCount, threads, smem>>>(map, p, sink);
        cudaEventRecord(e0);
        const int reps = 5;
        for (int rep = 0; rep < reps; ++rep) probe_kernel<<<prop.multiProcessorCount, threads, smem>>>(map, p, sink);
        cudaEventRecord(e1); cudaEventSynchronize(e1);
        float ms; cudaEventElapsedTime(&ms, e0, e1); ms /= reps;
        cudaError_t err = cudaGetLastError();
        double alg = (double)n * 4, moved = (double)N * 4 * p.bw * p.bh * 4.0 * p.n_tiles_x * p.n_tiles_y;
        printf("tile %dx%d box %dx%d rc %2d lds/px %2d cons_warps %2d smem %6zu: %.3f ms  alg %.0f GB/s  staged %.0f GB/s  %s\n", c.tw, c.th, c.bw, p.bh,
               c.rc, c.lds, c.warps, smem, ms, alg / ms / 1e6, moved / ms / 1e6, cudaGetErrorString(err));
    }
    return 0;
}
