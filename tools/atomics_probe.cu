// tools/atomics_probe.cu -- design input for the backward kernel: throughput of (1) global red.add.f32 with the
// scatter pattern of the bilinear backward (32 lanes -> 32 consecutive floats, 16 instrs per pixel-plane),
// (2) shared-memory fp32 atomic adds with the same pattern, (3) TMA reduce-add (cp.reduce.async.bulk.tensor) of tiles.
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include "../ml_gmpi_b200/csrc/tma_utils.cuh"
using namespace gmpi;

__global__ void __launch_bounds__(256) k_global_red(float* g, int planes, int W, int H) {
    // one thread per pixel of a 1024^2 image; per plane 16 reds to 4 channels x 2 rows x (x, x+1)
    const int px = blockIdx.x * 32 + (threadIdx.x & 31), py = blockIdx.y * 8 + (threadIdx.x >> 5);
    const size_t tex = (size_t)W * H;
    for (int i = 0; i < planes; ++i) {
        float* base = g + (size_t)i * 4 * tex + (size_t)py * W + px;
        const float v = 1e-3f * (i + 1);
#pragma unroll
        for (int c = 0; c < 4; ++c) {
            float* b = base + c * tex;
            atomicAdd(b, v); atomicAdd(b + 1, v); atomicAdd(b + W, v); atomicAdd(b + W + 1, v);
        }
    }
}

__global__ void __launch_bounds__(512) k_shared_red(float* out, int iters) {
    extern __shared__ float sm[];
    for (int i = threadIdx.x; i < 16384; i += blockDim.x) sm[i] = 0.f;
    __syncthreads();
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    long long t0 = clock64();
    for (int it = 0; it < iters; ++it) {
        float* b = sm + ((warp * 37 + it * 5) & 127) * 64 + lane;      // unit stride across lanes, rows vary
        const float v = 1e-3f;
#pragma unroll
        for (int c = 0; c < 4; ++c) {
            atomicAdd(b + c * 1024, v); atomicAdd(b + c * 1024 + 1, v); atomicAdd(b + c * 1024 + 72, v); atomicAdd(b + c * 1024 + 73, v);
        }
    }
    __syncthreads();
    long long t1 = clock64();
    if (threadIdx.x == 0) out[blockIdx.x] = (float)(t1 - t0);
    if (threadIdx.x == 1) out[1000 + blockIdx.x] = sm[5];
}

__global__ void __launch_bounds__(128) k_tma_reduce(const __grid_constant__ CUtensorMap map, int n_planes, int tiles_x, int tiles_y, int bw, int rows) {
    extern __shared__ __align__(1024) unsigned char smem[];
    float* buf = reinterpret_cast<float*>(smem);
    for (int i = threadIdx.x; i < bw * rows * 4; i += blockDim.x) buf[i] = 1e-3f;
    fence_proxy_async();
    __syncthreads();
    if (threadIdx.x == 0) {
        for (int t = blockIdx.x; t < tiles_x * tiles_y; t += gridDim.x) {
            const int x = (t % tiles_x) * 64, y = (t / tiles_x) * 30;
            for (int pl = 0; pl < n_planes; ++pl) {
                asm volatile("cp.reduce.async.bulk.tensor.4d.global.shared::cta.add.tile.bulk_group [%0, {%2, %3, %4, %5}], [%1];"
                             ::"l"(&map), "r"(smem_u32(buf)), "r"(x), "r"(0), "r"(y), "r"(pl) : "memory");
                asm volatile("cp.async.bulk.commit_group;" ::: "memory");
                asm volatile("cp.async.bulk.wait_group.read 4;" ::: "memory");
            }
        }
        asm volatile("cp.async.bulk.wait_group 0;" ::: "memory");
    }
}

int main() {
    int sms = 0;
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, 0);     // one CTA per SM
    const int N = 96, W = 1024, H = 1024;
    float* g; size_t n = (size_t)N * 4 * W * H;
    cudaMalloc(&g, n * 4 + (1 << 20)); cudaMemset(g, 0, n * 4);
    cudaEvent_t e0, e1; cudaEventCreate(&e0); cudaEventCreate(&e1); float ms;
    // (1) global reds
    dim3 grid((W - 32) / 32, (H - 8) / 8);
    k_global_red<<<grid, 256>>>(g, 8, W, H);
    cudaEventRecord(e0); k_global_red<<<grid, 256>>>(g, N, W, H); cudaEventRecord(e1); cudaEventSynchronize(e1);
    cudaEventElapsedTime(&ms, e0, e1);
    printf("global red.add.f32: %d planes x 1024^2 px x 16 reds: %.3f ms  (%.1f G lane-atomics/s) %s\n", N, ms, 16.0 * N * (W - 32) * (H - 8) / ms / 1e6, cudaGetErrorString(cudaGetLastError()));
    // (2) shared atomics
    float* out; cudaMalloc(&out, 8192 * 4);
    cudaFuncSetAttribute(k_shared_red, cudaFuncAttributeMaxDynamicSharedMemorySize, 65536);
    k_shared_red<<<sms, 512, 65536>>>(out, 2000); cudaDeviceSynchronize();
    float h[4]; cudaMemcpy(h, out, 16, cudaMemcpyDeviceToHost);
    printf("shared atomicAdd f32: 16 warps x 2000 iters x 16 instrs: %.0f cycles -> %.2f cycles per warp-instr per SM  %s\n", h[0], h[0] / (2000.0 * 16 * 16), cudaGetErrorString(cudaGetLastError()));
    // (3) TMA reduce-add
    CUtensorMap map;
    const int bw = 72, rows = 36;
    if (encode_plane_map(&map, g, MapElem{CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 4}, N, H, W, bw, rows) != 0) { printf("encode failed\n"); return 1; }
    cudaFuncSetAttribute(k_tma_reduce, cudaFuncAttributeMaxDynamicSharedMemorySize, bw * rows * 16);
    k_tma_reduce<<<sms, 128, bw * rows * 16>>>(map, 4, 16, 35, bw, rows);
    cudaEventRecord(e0); k_tma_reduce<<<sms, 128, bw * rows * 16>>>(map, N, 16, 35, bw, rows); cudaEventRecord(e1); cudaEventSynchronize(e1);
    cudaEventElapsedTime(&ms, e0, e1);
    printf("TMA reduce-add: %d planes x 560 tiles of %dx%dx4: %.3f ms (%.0f GB/s of tile bytes) %s\n", N, bw, rows, ms, (double)N * 560 * bw * rows * 16 / ms / 1e6, cudaGetErrorString(cudaGetLastError()));
    float hv[2]; cudaMemcpy(hv, g + (size_t)W * 100 + 100, 8, cudaMemcpyDeviceToHost); printf("sample %g %g\n", hv[0], hv[1]);
    return 0;
}
