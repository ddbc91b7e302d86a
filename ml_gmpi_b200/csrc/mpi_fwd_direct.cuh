// Forward, direct-gather variant: one thread = one output pixel, a warp = 32 consecutive x.  Taps are read straight from global
// memory through L1 (per channel a warp touches one or two 128-byte lines per tap row).  Works for every shape; the TMA-staged
// variant is the fast path.  Shared by the library's kernels (mpi_render.cu) and the uint8 kernels (mpi_u8.cu); the direct backward
// is in mpi_bwd_direct.cuh.
#pragma once
#include "mpi_common.cuh"
#include "mpi_kernel_keys.cuh"

namespace gmpi {

constexpr int kFwdTileW = 32;
constexpr int kFwdTileH = 8;

// kES: GMPI_EARLY_STOP, a pixel composites no further plane once |T| <= p.early_stop.
// (p by value: with a reference ptxas allocates the default kernel's registers differently.)  E: the MPI's element type.
template <bool kAlignCorners, bool kES, class E = float>
__device__ __forceinline__ void fwd_direct_body(const RenderParams p) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    PlaneConst* s_pc = reinterpret_cast<PlaneConst*>(smem_raw);

    const int v = blockIdx.z;
    const int m = __ldg(p.view2mpi + v);
    const int tid = threadIdx.y * kFwdTileW + threadIdx.x;
    float ev[3], zd[3];
    load_eye_z(p, v, ev, zd);
    const float eye0_z = __ldg(p.eye0 + 2);  // mpi.py:70 compares every distance with view 0's eye
    uint32_t flag = 0;
    for (int i = tid; i < p.N; i += kFwdTileW * kFwdTileH) {
        const float* dp = p.dhw + ((size_t)m * p.N + i) * 3;
        s_pc[i] = make_plane_const(dp, ev[2]);
        if (!(__ldg(dp) >= eye0_z)) flag |= GMPI_FLAG_PLANE_BEHIND_EYE;
    }
    __syncthreads();

    const int px = blockIdx.x * kFwdTileW + threadIdx.x;
    const int py = blockIdx.y * kFwdTileH + threadIdx.y;
    if (px < p.W && py < p.H) {
        const size_t img = (size_t)p.H * p.W;
        const size_t pix = (size_t)py * p.W + px;
        float qx, qy, qz;
        load_ray(p, v, px, py, img, qx, qy, qz);
        const RayConst rc = make_ray_const(qx, qy, qz, ev, zd);

        const int Ht = p.Ht, Wt = p.Wt;
        const float fWt = (float)Wt, fHt = (float)Ht;
        const float hsx = 0.5f * (float)(Wt - 1), hsy = 0.5f * (float)(Ht - 1);
        const size_t tex = (size_t)Ht * Wt;
        const bool check_last = (p.options & GMPI_CHECK_LAST_PLANE) != 0;
        const float tau = kES ? p.early_stop : 0.0f;

        float T = 1.0f, cr = 0.0f, cg = 0.0f, cb = 0.0f, cws = 0.0f;
#pragma unroll 2
        for (int i = 0; i < p.N; ++i) {
            const PlaneConst pc = s_pc[i];
            const PlaneChansT<E> plane = plane_chans<E>(p, m, i, tex);
            if (!kES && p.transmittance) p.transmittance[((size_t)v * p.N + i) * img + pix] = T;   // training: T_i for the backward sweep
            const TexCoord tc = plane_coord<kAlignCorners>(pc, rc, hsx, hsy, fWt, fHt);
            if (check_last && i == p.N - 1) {
                if (!(tc.u >= -1.0f && tc.u <= 1.0f && tc.v >= -1.0f && tc.v <= 1.0f)) flag |= GMPI_FLAG_LAST_PLANE_OOB;
            }
            if (coord_hits(tc.ix, tc.iy, fWt, fHt) && !(kES && fabsf(T) <= tau)) {
                const Taps t = make_taps(tc.ix, tc.iy, Ht, Wt);
                const float r = tap4(plane.c[0], t);
                const float g = tap4(plane.c[1], t);
                const float b = tap4(plane.c[2], t);
                const float a = tap4(plane.c[3], t);
                const float w = a * T;                                   // mpi.py:423
                cr = fmaf(w, r, cr);                                     // mpi.py:430
                cg = fmaf(w, g, cg);
                cb = fmaf(w, b, cb);
                cws = fmaf(w, tc.scale, cws);                            // depth_i = scale * (ray.z_dir), :150
                T *= (1.0f - a) + 1e-10f;                                // mpi.py:421
            }
        }
        const float dep = cws * rc.dz;
        if (p.options & GMPI_COLOR_MINUS1_1) {                           // mpi_renderer.py:467
            cr = fmaf(2.0f, cr, -1.0f);
            cg = fmaf(2.0f, cg, -1.0f);
            cb = fmaf(2.0f, cb, -1.0f);
        }
        store_pixel(p, v, img, pix, cr, cg, cb, dep);
    }
    if (flag) atomicOr(p.flags, flag);
}

// The direct forward kernels by key (KeyTraits): fp32, fp16 and uint8 MPIs, early stop.
template <uint32_t K>
__global__ void __launch_bounds__(kFwdTileW* kFwdTileH) mpi_fwd_direct_kernel(const RenderParams p) {
    using T = KeyTraits<K>;
    static_assert((K & (kKeyStaged | kKeyBwd | kKeySkip | kKeyFac | kKeyEmit)) == 0, "a direct forward key");
    fwd_direct_body<T::kAlignCorners, T::kES, typename T::Elem>(p);
}

}  // namespace gmpi
