// The kernels behind the library's test hooks (the gmpi_debug_* entry points of mpi_render.cu, its only includer): the texel
// coordinates of the direct and the pixel-pair path, the division the kernels use, and the rays of a camera matrix.
#pragma once
#include "mpi_common.cuh"
#include "mpi_fwd_staged.cuh"

namespace gmpi {

// Texel coordinates.
template <bool kAlignCorners>
__global__ void mpi_debug_coords_kernel(const int32_t* view2mpi, const float* dhw, const float* ray_dir,
                                        const float* eye, float* out, int V, int N, int Ht, int Wt, int H, int W) {
    const size_t img = (size_t)H * W;
    const size_t pix = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    const int v = blockIdx.y;
    if (pix >= img) return;
    const int m = view2mpi[v];
    const float* e = eye + 3 * v;
    const float ev[3] = {e[0], e[1], e[2]};
    const float zd[3] = {0.f, 0.f, 1.f};
    const float* rd = ray_dir + (size_t)v * 3 * img + pix;
    const RayConst rc = make_ray_const(rd[0], rd[img], rd[2 * img], ev, zd);
    const float hsx = 0.5f * (float)(Wt - 1), hsy = 0.5f * (float)(Ht - 1);
    for (int i = 0; i < N; ++i) {
        const PlaneConst pc = make_plane_const(dhw + ((size_t)m * N + i) * 3, ev[2]);
        const TexCoord tc = plane_coord<kAlignCorners>(pc, rc, hsx, hsy, (float)Wt, (float)Ht);
        out[(((size_t)v * N + i) * 2 + 0) * img + pix] = tc.ix;
        out[(((size_t)v * N + i) * 2 + 1) * img + pix] = tc.iy;
    }
}

// Test hook for the pixel-pair coordinate path of the staged kernel: pixels 2k, 2k+1 of a row form a pair (both of the staged
// kernel's pairs per thread hold it).
template <bool kAlignCorners>
__global__ void mpi_debug_coords_packed_kernel(const int32_t* view2mpi, const float* dhw, const float* ray_dir,
                                               const float* eye, float* out, int V, int N, int Ht, int Wt, int H, int W) {
    const size_t img = (size_t)H * W;
    const size_t pair = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    const int v = blockIdx.y;
    if (pair * 2 + 1 >= img) return;
    const int m = view2mpi[v];
    const float* e = eye + 3 * v;
    const float ev[3] = {e[0], e[1], e[2]};
    const float zd[3] = {0.f, 0.f, 1.f};
    RayConst rc[kPix];
    for (int q = 0; q < kPix; ++q) {
        const float* rd = ray_dir + (size_t)v * 3 * img + pair * 2 + (q & 1);
        rc[q] = make_ray_const(rd[0], rd[img], rd[2 * img], ev, zd);
    }
    RayPairs rp;
    pack_ray_pairs(rc, rp);
    const float hsx = 0.5f * (float)(Wt - 1), hsy = 0.5f * (float)(Ht - 1);
    for (int i = 0; i < N; ++i) {
        const PlaneConst pc = make_plane_const(dhw + ((size_t)m * N + i) * 3, ev[2]);
        CoordPairs c;
        coords_pairs<kAlignCorners>(pc, rp, splat(rc[0].ex2), splat(rc[0].ey2), splat(hsx), splat(hsy), (float)Wt, (float)Ht, c);
        float* o = out + (((size_t)v * N + i) * 2) * img + pair * 2;
        o[0] = c.ix[0].x; o[1] = c.ix[0].y; o[img] = c.iy[0].x; o[img + 1] = c.iy[0].y;
    }
}

__global__ void mpi_debug_division_kernel(const float* a, const float* b, float* out_fast, float* out_ieee, size_t n) {
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
        const float x = a[i], y = b[i];
        out_fast[i] = in_safe_range(y) && (x == 0.0f || in_safe_range(x)) ? div_by_rcp(x, y, __frcp_rn(y)) : __fdiv_rn(x, y);
        out_ieee[i] = __fdiv_rn(x, y);
    }
}

__global__ void mpi_debug_cam_rays_kernel(const float* __restrict__ cam, float* __restrict__ ray_dir, int V, int H, int W) {
    const size_t img = (size_t)H * W;
    const size_t pix = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    const int v = blockIdx.y;
    if (pix >= img) return;
    float rx, ry, rz;
    cam_ray(cam + 16 * (size_t)v, (int)(pix % W), (int)(pix / W), H, W, rx, ry, rz);
    float* o = ray_dir + (size_t)v * 3 * img + pix;
    o[0] = rx; o[img] = ry; o[2 * img] = rz;
}

}  // namespace gmpi
