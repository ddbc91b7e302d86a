// tools/l2_reduce_probe.cu -- round-2 design input for the backward kernel: what bounds gradient accumulation into a
// 96 x 4 x 1024^2 fp32 buffer (1.61 GB, far larger than L2, so every variant pays the read-modify-write through DRAM)?
//   P0  plain coalesced stores of every element once            (write bandwidth reference)
//   P1  red.global.add.f32, dense: every element exactly once, a warp = 32 consecutive floats
//   P2  red.global.add.v4.f32, dense: a lane = 4 consecutive floats
//   P3  red.global.add.f32, sparse: same instruction count as P1 but only every 8th lane active (sector- or lane-bound?)
//   P4  P1 pattern issued 4x per element (the 16-tap scatter of the current kernel touches every texel 4x per channel)
//   P5  TMA reduce-add of disjoint 64x32x4 boxes, 1 issuing thread per SM, up to 8 boxes in flight
//   S*  shared-memory accumulation cost per warp instruction: CAS-loop atomicAdd(float), red.shared.add.f32 (PTX),
//       integer atomicAdd, and the non-atomic LDS+FADD+STS sequence
// Build: nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o tools/l2_reduce_probe tools/l2_reduce_probe.cu
#include <cstdio>
#include <cstdlib>
#include "../ml_gmpi_b200/csrc/tma_utils.cuh"
using namespace gmpi;

constexpr int N = 96, W = 1024, H = 1024;
constexpr size_t kElems = (size_t)N * 4 * W * H;

__global__ void __launch_bounds__(256) k_store(float* g, size_t n) {
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) g[i] = 1e-3f;
}
__global__ void __launch_bounds__(256) k_red_dense(float* g, size_t n, int repeat) {
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x)
        for (int r = 0; r < repeat; ++r) asm volatile("red.global.add.f32 [%0], %1;" ::"l"(g + i), "f"(1e-3f) : "memory");
}
__global__ void __launch_bounds__(256) k_red_v4(float* g, size_t n4) {
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += (size_t)gridDim.x * blockDim.x)
        asm volatile("red.global.add.v4.f32 [%0], {%1, %1, %1, %1};" ::"l"(g + 4 * i), "f"(1e-3f) : "memory");
}
__global__ void __launch_bounds__(256) k_red_sparse(float* g, size_t n) {
    const bool on = (threadIdx.x & 7) == 0;
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x)
        if (on) asm volatile("red.global.add.f32 [%0], %1;" ::"l"(g + i), "f"(1e-3f) : "memory");
}
__global__ void __launch_bounds__(128) k_tma_reduce(const __grid_constant__ CUtensorMap map, int n_planes, int tiles_x, int tiles_y, int bw, int rows) {
    extern __shared__ __align__(1024) unsigned char smem[];
    float* buf = reinterpret_cast<float*>(smem);
    for (int i = threadIdx.x; i < bw * rows * 4; i += blockDim.x) buf[i] = 1e-3f;
    fence_proxy_async();
    __syncthreads();
    if (threadIdx.x == 0) {
        for (int t = blockIdx.x; t < tiles_x * tiles_y; t += gridDim.x) {
            const int x = (t % tiles_x) * bw, y = (t / tiles_x) * rows;
            for (int pl = 0; pl < n_planes; ++pl) {
                asm volatile("cp.reduce.async.bulk.tensor.4d.global.shared::cta.add.tile.bulk_group [%0, {%2, %3, %4, %5}], [%1];"
                             ::"l"(&map), "r"(smem_u32(buf)), "r"(x), "r"(0), "r"(y), "r"(pl) : "memory");
                asm volatile("cp.async.bulk.commit_group;" ::: "memory");
                asm volatile("cp.async.bulk.wait_group.read 8;" ::: "memory");
            }
        }
        asm volatile("cp.async.bulk.wait_group 0;" ::: "memory");
    }
}

// shared-memory accumulate variants: 16 warps, each iteration 16 warp instructions on unit-stride addresses
template <int MODE>
__global__ void __launch_bounds__(512) k_shared(float* out, int iters) {
    extern __shared__ float sm[];
    for (int i = threadIdx.x; i < 16384; i += blockDim.x) sm[i] = 0.f;
    __syncthreads();
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    long long t0 = clock64();
    for (int it = 0; it < iters; ++it) {
        float* b = sm + ((warp * 37 + it * 5) & 127) * 64 + lane;
        const float v = 1e-3f;
#pragma unroll
        for (int c = 0; c < 4; ++c) {
#pragma unroll
            for (int k = 0; k < 4; ++k) {
                float* a = b + c * 1024 + (k & 1) + (k >> 1) * 72;
                if (MODE == 0) atomicAdd(a, v);
                else if (MODE == 1) asm volatile("red.shared.add.f32 [%0], %1;" ::"r"(smem_u32(a)), "f"(v) : "memory");
                else if (MODE == 2) atomicAdd(reinterpret_cast<int*>(a), 3);
                else { *a = *a + v; __syncwarp(); }
            }
        }
    }
    __syncthreads();
    long long t1 = clock64();
    if (threadIdx.x == 0) out[blockIdx.x] = (float)(t1 - t0);
    if (threadIdx.x == 1) out[1000 + blockIdx.x] = sm[5];
}

int main() {
    int sms = 0;
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, 0);     // one CTA per SM
    float* g;
    cudaMalloc(&g, kElems * 4 + (1 << 20));
    cudaMemset(g, 0, kElems * 4);
    cudaEvent_t e0, e1; cudaEventCreate(&e0); cudaEventCreate(&e1); float ms;
    auto timeit = [&](const char* name, auto launch, double elems) {
        launch();                                   // warm-up
        cudaEventRecord(e0); launch(); cudaEventRecord(e1); cudaEventSynchronize(e1);
        cudaEventElapsedTime(&ms, e0, e1);
        printf("%-58s %.3f ms  %.0f G elem/s  %s\n", name, ms, elems / ms / 1e6, cudaGetErrorString(cudaGetLastError()));
    };
    const int grid = sms * 8;
    timeit("P0 st.global.f32 dense, every element once", [&] { k_store<<<grid, 256>>>(g, kElems); }, (double)kElems);
    cudaMemset(g, 0, kElems * 4);
    timeit("P1 red.global.add.f32 dense, every element once", [&] { k_red_dense<<<grid, 256>>>(g, kElems, 1); }, (double)kElems);
    timeit("P2 red.global.add.v4.f32 dense, every element once", [&] { k_red_v4<<<grid, 256>>>(g, kElems / 4); }, (double)kElems);
    timeit("P3 red.global.add.f32 sparse (1 lane in 8), same instrs as P1", [&] { k_red_sparse<<<grid, 256>>>(g, kElems); }, (double)kElems / 8);
    timeit("P4 red.global.add.f32 dense, every element 4x back to back", [&] { k_red_dense<<<grid, 256>>>(g, kElems, 4); }, 4.0 * kElems);
    {
        CUtensorMap map;
        const int bw = 64, rows = 32;
        if (encode_plane_map(&map, g, MapElem{CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 4}, N, H, W, bw, rows) != 0) { printf("encode failed\n"); return 1; }
        cudaFuncSetAttribute(k_tma_reduce, cudaFuncAttributeMaxDynamicSharedMemorySize, bw * rows * 16);
        timeit("P5 TMA reduce-add, disjoint 64x32x4 boxes, every element once",
               [&] { k_tma_reduce<<<sms, 128, bw * rows * 16>>>(map, N, W / bw, H / rows, bw, rows); }, (double)kElems);
    }
    {
        CUtensorMap map;
        const int bw = 72, rows = 36;       // overlapping, as a footprint-fitted gradient box would be (origin step 64x30)
        if (encode_plane_map(&map, g, MapElem{CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 4}, N, H, W, bw, rows) != 0) { printf("encode failed\n"); return 1; }
        cudaFuncSetAttribute(k_tma_reduce, cudaFuncAttributeMaxDynamicSharedMemorySize, bw * rows * 16);
        timeit("P5b TMA reduce-add, 72x36x4 boxes stepping by 72x36 (unaligned rows)",
               [&] { k_tma_reduce<<<sms, 128, bw * rows * 16>>>(map, N, W / bw, H / rows, bw, rows); }, (double)N * (W / bw) * (H / rows) * bw * rows * 4);
    }
    float* out; cudaMalloc(&out, 8192 * 4);
    float h[1];
    auto shared = [&](const char* name, auto kern) {
        cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, 65536);
        kern<<<sms, 512, 65536>>>(out, 2000); cudaDeviceSynchronize();
        cudaMemcpy(h, out, 4, cudaMemcpyDeviceToHost);
        printf("%-58s %.2f cycles per warp instruction per SM  %s\n", name, h[0] / (2000.0 * 16 * 16), cudaGetErrorString(cudaGetLastError()));
    };
    shared("S0 shared atomicAdd(float) (CAS loop)", k_shared<0>);
    shared("S1 red.shared.add.f32 (PTX)", k_shared<1>);
    shared("S2 shared atomicAdd(int)", k_shared<2>);
    shared("S3 shared LDS+FADD+STS (non-atomic)", k_shared<3>);
    return 0;
}
