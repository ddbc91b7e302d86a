// Kernels behind LightRenderer (gmpi/core/light_renderer.py), the lighting augmentation applied to the MPI right before the
// render call during training (train.py:534-541,702-709) -- SURVEY.md 8(f) row N3:
//
//   compute_depth (light_renderer.py:82-100): the same over-composite as the renderer, on the UN-warped alpha:
//       T_i = prod_{j<i}(1 - a_j + 1e-10),  depth = sum_i a_i T_i d_i          -> [M,1,Ht,Wt]
//     The reference materialises [M,N+1,1,H,W] (cat), its cumprod, the weights and their product with plane_ds: ~5 full-size
//     tensors.  Here: one streaming pass, 4 B read per texel-plane, float4 per thread, nothing materialised; the training
//     variant also stores T_i (what the backward needs).
//   render's last step (light_renderer.py:190-199): new_rgb = clip(rgb * shading, 0, 1), alpha unchanged, cat -> a new MPI:
//     one fused pass (read 16 B, write 16 B per texel-plane) instead of mul + clip + cat.
//
// Both are pure HBM streams: per-texel arithmetic, no sampling, no scatter.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace gmpi {

struct AlphaView {          // alpha of plane i of MPI m at base[m * mpi_stride + i * plane_stride + texel]  (strides in floats)
    const float* base;
    long long mpi_stride, plane_stride;
};

// One thread = four consecutive texels.  kSaveT: training forward (stores T_i, [M,N,Ht*Wt]).
template <bool kSaveT>
__global__ void __launch_bounds__(256)
mpi_alpha_depth_fwd_kernel(AlphaView a, const float* __restrict__ plane_d, float* __restrict__ depth, float* __restrict__ trans,
                           int N, long long tex4) {
    const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const int m = blockIdx.y;
    if (t >= tex4) return;
    const float4* ap = reinterpret_cast<const float4*>(a.base + (long long)m * a.mpi_stride) + t;
    const long long ps4 = a.plane_stride / 4;
    float4* tp = kSaveT ? reinterpret_cast<float4*>(trans + (long long)m * N * tex4 * 4) + t : nullptr;
    float4 T = make_float4(1.f, 1.f, 1.f, 1.f), acc = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll 4
    for (int i = 0; i < N; ++i) {
        const float4 al = __ldcs(ap + (long long)i * ps4);
        const float d = __ldg(plane_d + i);
        if (kSaveT) __stcs(tp + (long long)i * tex4, T);
        acc.x = fmaf(al.x * T.x, d, acc.x); acc.y = fmaf(al.y * T.y, d, acc.y);          // weights * plane_ds, summed (:88,:98)
        acc.z = fmaf(al.z * T.z, d, acc.z); acc.w = fmaf(al.w * T.w, d, acc.w);
        T.x *= (1.0f - al.x) + 1e-10f; T.y *= (1.0f - al.y) + 1e-10f;                    // cumprod of (1 - a + 1e-10) (:86-88)
        T.z *= (1.0f - al.z) + 1e-10f; T.w *= (1.0f - al.w) + 1e-10f;
    }
    reinterpret_cast<float4*>(depth + (long long)m * tex4 * 4)[t] = acc;
}

// d depth / d alpha_i = T_i (q_i - R_i) with q_i = G d_i and R_{i-1} = a_i q_i + (1 - a_i + 1e-10) R_i, R_{N-1} = 0: autograd's
// cumprod_backward without the division by (1 - a_i + 1e-10) (see the renderer's backward).  Back to front, T_i from the forward.
__global__ void __launch_bounds__(256)
mpi_alpha_depth_bwd_kernel(AlphaView a, const float* __restrict__ plane_d, const float* __restrict__ trans, const float* __restrict__ g_depth,
                           float* __restrict__ g_alpha, long long g_mpi_stride, long long g_plane_stride, int N, long long tex4) {
    const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const int m = blockIdx.y;
    if (t >= tex4) return;
    const float4* ap = reinterpret_cast<const float4*>(a.base + (long long)m * a.mpi_stride) + t;
    const long long ps4 = a.plane_stride / 4;
    const float4* tp = reinterpret_cast<const float4*>(trans + (long long)m * N * tex4 * 4) + t;
    float4* gp = reinterpret_cast<float4*>(g_alpha + (long long)m * g_mpi_stride) + t;
    const long long gs4 = g_plane_stride / 4;
    const float4 G = reinterpret_cast<const float4*>(g_depth + (long long)m * tex4 * 4)[t];
    float4 R = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll 4
    for (int i = N - 1; i >= 0; --i) {
        const float4 al = __ldcs(ap + (long long)i * ps4), T = __ldcs(tp + (long long)i * tex4);
        const float d = __ldg(plane_d + i);
        float4 g;
        g.x = T.x * (G.x * d - R.x); g.y = T.y * (G.y * d - R.y); g.z = T.z * (G.z * d - R.z); g.w = T.w * (G.w * d - R.w);
        __stcs(gp + (long long)i * gs4, g);
        R.x = fmaf(al.x, G.x * d, ((1.0f - al.x) + 1e-10f) * R.x); R.y = fmaf(al.y, G.y * d, ((1.0f - al.y) + 1e-10f) * R.y);
        R.z = fmaf(al.z, G.z * d, ((1.0f - al.z) + 1e-10f) * R.z); R.w = fmaf(al.w, G.w * d, ((1.0f - al.w) + 1e-10f) * R.w);
    }
}

// torch.clip(x, 0, 1): a NaN stays NaN (fmaxf alone returns 0 for it, which would hide a diverging colour in the shaded MPI);
// every other value takes the same fminf(fmaxf) as torch's clamp, so the result is bit for bit torch's.
__device__ __forceinline__ float clip01(float x) { return isnan(x) ? x : fminf(fmaxf(x, 0.0f), 1.0f); }

// out[m,i,c] = clip(rgba[m,i,c] * shade[m], 0, 1) for c < 3, out[m,i,3] = rgba[m,i,3]   (light_renderer.py:190-199)
// grid: (tex4 blocks, N, M); one thread = four texels of one plane, all four channels.
__global__ void __launch_bounds__(256)
mpi_apply_shading_fwd_kernel(const float* __restrict__ rgba, const float* __restrict__ shade, float* __restrict__ out, int N, long long tex4) {
    const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= tex4) return;
    const int i = blockIdx.y, m = blockIdx.z;
    const float4 s = reinterpret_cast<const float4*>(shade + (long long)m * tex4 * 4)[t];
    const long long plane = ((long long)m * N + i) * 4 * tex4;
    const float4* in = reinterpret_cast<const float4*>(rgba) + plane + t;
    float4* o = reinterpret_cast<float4*>(out) + plane + t;
#pragma unroll
    for (int c = 0; c < 3; ++c) {
        const float4 x = __ldcs(in + c * tex4);
        __stcs(o + c * tex4, make_float4(clip01(x.x * s.x), clip01(x.y * s.y), clip01(x.z * s.z), clip01(x.w * s.w)));
    }
    __stcs(o + 3 * tex4, __ldcs(in + 3 * tex4));
}

// Gradient of the above: g_rgba[c<3] = g_out * shade where 0 <= rgb * shade <= 1 (torch.clip passes the gradient on the closed
// interval), g_rgba[3] = g_out[3]; g_shade[m] = sum over planes and colour channels of g_out * rgb under the same mask.
// grid: (tex4 blocks, M); a thread walks the N planes of its four texels, so g_shade needs no atomics.
__global__ void __launch_bounds__(256)
mpi_apply_shading_bwd_kernel(const float* __restrict__ rgba, const float* __restrict__ shade, const float* __restrict__ g_out,
                             float* __restrict__ g_rgba, float* __restrict__ g_shade, int N, long long tex4) {
    const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= tex4) return;
    const int m = blockIdx.y;
    const float4 s = reinterpret_cast<const float4*>(shade + (long long)m * tex4 * 4)[t];
    float4 gs = make_float4(0.f, 0.f, 0.f, 0.f);
    for (int i = 0; i < N; ++i) {
        const long long plane = ((long long)m * N + i) * 4 * tex4;
        const float4* in = reinterpret_cast<const float4*>(rgba) + plane + t;
        const float4* go = reinterpret_cast<const float4*>(g_out) + plane + t;
        float4* gi = reinterpret_cast<float4*>(g_rgba) + plane + t;
#pragma unroll
        for (int c = 0; c < 3; ++c) {
            const float4 x = __ldcs(in + c * tex4), g = __ldcs(go + c * tex4);
            float4 r;
            float p;
            p = x.x * s.x; r.x = (p >= 0.0f && p <= 1.0f) ? g.x : 0.0f;
            p = x.y * s.y; r.y = (p >= 0.0f && p <= 1.0f) ? g.y : 0.0f;
            p = x.z * s.z; r.z = (p >= 0.0f && p <= 1.0f) ? g.z : 0.0f;
            p = x.w * s.w; r.w = (p >= 0.0f && p <= 1.0f) ? g.w : 0.0f;
            gs.x = fmaf(r.x, x.x, gs.x); gs.y = fmaf(r.y, x.y, gs.y); gs.z = fmaf(r.z, x.z, gs.z); gs.w = fmaf(r.w, x.w, gs.w);
            __stcs(gi + c * tex4, make_float4(r.x * s.x, r.y * s.y, r.z * s.z, r.w * s.w));
        }
        __stcs(gi + 3 * tex4, __ldcs(go + 3 * tex4));
    }
    reinterpret_cast<float4*>(g_shade + (long long)m * tex4 * 4)[t] = gs;
}

}  // namespace gmpi
