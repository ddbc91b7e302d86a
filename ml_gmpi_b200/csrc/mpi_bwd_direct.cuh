// The direct backward kernels, the counterpart of mpi_fwd_direct.cuh: taps read and gradients scattered straight through global
// memory.  Any shape, no saved state; the box kernel (mpi_bwd_box.cuh) is the fast path.  Launched by mpi_render.cu.
#pragma once
#include "mpi_common.cuh"
#include "mpi_bwd_box.cuh"
#include "mpi_kernel_keys.cuh"

namespace gmpi {

// ------------------------------------------------------------------------------------------
// Backward, direct variant.
//   pass A (front to back, alpha only): T_i = prod_{j<i}(1 - a_j + 1e-10), stashed per thread in
//           shared memory ([plane][thread], conflict free).
//   pass B (back to front, all channels): R_{i-1} = a_i q_i + s_i R_i with R_{N-1} = 0,
//           q_i = G.rgb_i + Gd*depth_i, s_i = 1 - a_i + 1e-10, and
//             dL/d rgb_i = G * a_i T_i
//             dL/d a_i   = T_i (q_i - R_i)
//           which equals autograd's  T_i q_i - (sum_{k>i} a_k q_k P_k)/s_i  (cumprod_backward)
//           without the division by s_i (1e-10 when a_i == 1) and without cancellation.
//           The four bilinear weights scatter each value with red.global.add.f32.
// kDet: the deterministic backward's variant, which adds each contribution to the int64 sums of `da` instead (det_add).
// ------------------------------------------------------------------------------------------
template <bool kAlignCorners, bool kDet>
__device__ __forceinline__ void bwd_direct_body(const RenderParams p, const int tile_w, const int tile_h, const DetAcc da) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    PlaneConst* s_pc = reinterpret_cast<PlaneConst*>(smem_raw);
    const int nthreads = tile_w * tile_h;
    float* s_T = reinterpret_cast<float*>(smem_raw + sizeof(PlaneConst) * p.N);   // [N][nthreads]

    const int v = blockIdx.z;
    const int m = __ldg(p.view2mpi + v);
    const int tid = threadIdx.y * tile_w + threadIdx.x;
    const float* e = p.eye + 3 * v;
    for (int i = tid; i < p.N; i += nthreads) {
        s_pc[i] = make_plane_const(p.dhw + ((size_t)m * p.N + i) * 3, __ldg(e + 2));
    }
    __syncthreads();

    const int px = blockIdx.x * tile_w + threadIdx.x;
    const int py = blockIdx.y * tile_h + threadIdx.y;
    if (px >= p.W || py >= p.H) return;

    const size_t img = (size_t)p.H * p.W;
    const size_t pix = (size_t)py * p.W + px;
    const float* rd = p.ray_dir + (size_t)v * 3 * img + pix;
    const float ev[3] = {__ldg(e), __ldg(e + 1), __ldg(e + 2)};
    const float zd[3] = {__ldg(p.z_dir + 3 * v), __ldg(p.z_dir + 3 * v + 1), __ldg(p.z_dir + 3 * v + 2)};
    const RayConst rc = make_ray_const(__ldg(rd), __ldg(rd + img), __ldg(rd + 2 * img), ev, zd);

    const int Ht = p.Ht, Wt = p.Wt, N = p.N;
    const float fWt = (float)Wt, fHt = (float)Ht;
    const float hsx = 0.5f * (float)(Wt - 1), hsy = 0.5f * (float)(Ht - 1);
    const size_t tex = (size_t)Ht * Wt;

    float gscale = (p.options & GMPI_COLOR_MINUS1_1) ? 2.0f : 1.0f;
    const float* gc = p.g_color + (size_t)v * 3 * img + pix;
    const float G0 = gscale * __ldg(gc), G1 = gscale * __ldg(gc + img), G2 = gscale * __ldg(gc + 2 * img);
    const float Gd = p.g_depth ? __ldg(p.g_depth + (size_t)v * img + pix) : 0.0f;
    const float Gdz = Gd * rc.dz;   // depth_i = scale_i * dz
    DetUnit ua{}, urgb{};
    if constexpr (kDet) {
        ua = det_unit(__uint_as_float(__ldg(da.bounds)), da.k_a);
        urgb = det_unit(0.5f * __uint_as_float(__ldg(da.bounds + 1)), da.k_rgb);
    }

    // pass A
    float T = 1.0f;
    for (int i = 0; i < N; ++i) {
        s_T[(size_t)i * nthreads + tid] = T;
        const TexCoord tc = plane_coord<kAlignCorners>(s_pc[i], rc, hsx, hsy, fWt, fHt);
        if (coord_hits(tc.ix, tc.iy, fWt, fHt)) {
            const Taps t = make_taps(tc.ix, tc.iy, Ht, Wt);
            const float a = tap4(plane_chans(p, m, i, tex).c[3], t);
            T *= (1.0f - a) + 1e-10f;
        }
    }
    // pass B
    float R = 0.0f;
    for (int i = N - 1; i >= 0; --i) {
        const TexCoord tc = plane_coord<kAlignCorners>(s_pc[i], rc, hsx, hsy, fWt, fHt);
        if (!coord_hits(tc.ix, tc.iy, fWt, fHt)) continue;
        const Taps t = make_taps(tc.ix, tc.iy, Ht, Wt);
        const PlaneChans plane = plane_chans(p, m, i, tex);
        const float r = tap4(plane.c[0], t);
        const float g = tap4(plane.c[1], t);
        const float b = tap4(plane.c[2], t);
        const float a = tap4(plane.c[3], t);
        const float Ti = s_T[(size_t)i * nthreads + tid];
        const float q = fmaf(G0, r, fmaf(G1, g, fmaf(G2, b, Gdz * tc.scale)));
        const float w = a * Ti;
        const float gv[4] = {G0 * w, G1 * w, G2 * w, Ti * (q - R)};
        R = fmaf(a, q, ((1.0f - a) + 1e-10f) * R);
        const GradChans gp = grad_chans(p, m, i, tex);
#pragma unroll
        for (int c = 0; c < 4; ++c) {
            float* gch = gp.c[c];
            if constexpr (kDet) {
                const DetUnit& u = c == 3 ? ua : urgb;
                if (t.w00 != 0.0f) det_add(da, u, gch + t.o00, gv[c] * t.w00);
                if (t.w01 != 0.0f) det_add(da, u, gch + t.o01, gv[c] * t.w01);
                if (t.w10 != 0.0f) det_add(da, u, gch + t.o10, gv[c] * t.w10);
                if (t.w11 != 0.0f) det_add(da, u, gch + t.o11, gv[c] * t.w11);
            } else {
                if (t.w00 != 0.0f) atomicAdd(gch + t.o00, gv[c] * t.w00);
                if (t.w01 != 0.0f) atomicAdd(gch + t.o01, gv[c] * t.w01);
                if (t.w10 != 0.0f) atomicAdd(gch + t.o10, gv[c] * t.w10);
                if (t.w11 != 0.0f) atomicAdd(gch + t.o11, gv[c] * t.w11);
            }
        }
    }
}

// The direct backward kernels by key (KeyTraits), and the deterministic ones (kKeyDet), which take the DetAcc too.
template <uint32_t K>
__global__ void __launch_bounds__(128)
mpi_bwd_direct_kernel(const RenderParams p, const int tile_w, const int tile_h) {
    static_assert((K & ~kKeyAC) == kKeyBwd, "a direct backward key");
    bwd_direct_body<KeyTraits<K>::kAlignCorners, false>(p, tile_w, tile_h, DetAcc{});
}

template <uint32_t K>
__global__ void __launch_bounds__(128)
mpi_bwd_direct_det_kernel(const RenderParams p, const int tile_w, const int tile_h, const DetAcc da) {
    static_assert((K & ~kKeyAC) == (kKeyBwd | kKeyDet), "a deterministic direct backward key");
    bwd_direct_body<KeyTraits<K>::kAlignCorners, true>(p, tile_w, tile_h, da);
}

}  // namespace gmpi
