// Backward, TMA-staged persistent kernel with a tile-local gradient box: d(sum(color*g_color) + sum(depth*g_depth)) / d rgba.
//
// Planes are walked BACK TO FRONT with the forward's tile / ring / producer machinery (mpi_fwd_staged.cuh).  The forward, run
// in training mode, saved the transmittance T_i in front of every plane ([V,N,H,W]); with it one sweep suffices:
//     q_i = G.rgb_i + G_d*depth_i          d_i = q_i - R_i            (R_{N-1} = 0)
//     dL/d rgb_i = G * a_i * T_i           dL/d a_i = T_i * d_i       R_{i-1} = R_i + a_i * d_i
// which is autograd's  T_i q_i - (sum_{k>i} a_k q_k P_k) / (1 - a_i + 1e-10)  (cumprod_backward) without the division
// (1e-10 when a_i == 1) and without cancellation; grid_sampler_2d_backward then scatters every value through the four bilinear
// weights.
//
// Where the scatter goes (round 2).  Round 1 issued 16 red.global.add.f32 per (pixel, plane): 46 M REDG warp instructions per
// view, each wrapped in BSSY/BRA/BSYNC when predicated, 64-bit address arithmetic, shuffles for tap hand-over -- 900 SASS
// instructions per thread and plane.  Shared-memory fp32 atomics are a CAS loop, native INTEGER shared atomics are one
// instruction, and a dense, coalesced red.global of the finished sums is bound only by the DRAM read-modify-write of the
// gradient.  Hence:
//   * every (tile, plane) has a GRADIENT BOX in shared memory with exactly the layout of the staged plane box
//     ([row][channel][x], same index as the taps);
//   * consumers add their 16 contributions per pixel with `red.shared.add.s32` on FIXED-POINT values: c * 2^(26-e) rounded to
//     nearest (three FMAs against magic constants, no F2I), where 2^e bounds every contribution of the tile (computed from the
//     tile's upstream gradients, see tile_scale_exponent).  26 bits per contribution relative to that bound, exact (order
//     independent) integer sums: more repeatable than fp32 atomics, a few 1e-6 of the largest gradient in error;
//   * three FLUSHER warps convert a finished box to fp32 and add it to g_rgba with coalesced `red.global.add.v4.f32`
//     (skipping all-zero quads and texels outside the texture) and re-zero it, while the consumers fill the other box.
// Out-of-texture taps need no predication: they land in box cells that lie outside the texture, which the flush drops
// (padding_mode="zeros").  A warp whose footprints do not all lie inside the staged box (non-projective rays, oversized
// footprints, planes outside the exact-division range) samples global memory and scatters with red.global.add.f32 directly,
// as the direct kernel does: results never depend on the producer's footprint estimate.
#pragma once
#include "mpi_fwd_staged.cuh"

namespace gmpi {

constexpr int kBwdConsWarps = 12, kBwdFlushWarps = 3;
constexpr int kBwdTileH = kPairs * kBwdConsWarps;                                   // 64 x 24 pixel tiles
constexpr int kBwdConsThreads = kBwdConsWarps * 32;
constexpr int kBwdThreads = (kBwdConsWarps + 1 + kBwdFlushWarps) * 32;              // 16 warps: 12 consumers, producer, 3 flushers
constexpr int kBwdStages = 2, kBwdBoxes = 2;
constexpr int kBwdMaxBH = (((kBwdTileH * 5) / 4 + 6 + kRowsPerOp - 1) / kRowsPerOp) * kRowsPerOp;
constexpr int kBwdPlaneFloats = kMaxBW * kBwdMaxBH * 4;
constexpr int kBwdTFloats = kTileW * kBwdTileH;
constexpr int kBwdStride = kBwdPlaneFloats + kBwdTFloats;
constexpr size_t kBwdSmem = (size_t)(kBwdStages * kBwdStride + kBwdBoxes * kBwdPlaneFloats) * 4 + (size_t)kMaxPlanesStaged * 32;
static_assert(kBwdSmem + 1024 <= 227 * 1024, "backward ring + gradient boxes + plane table must fit one SM");

struct BwdRing {
    static constexpr int kTileRows = kBwdTileH, kRingStages = kBwdStages, kBoxMaxH = kBwdMaxBH;
    static constexpr int kPlaneFloats = kBwdPlaneFloats, kStride = kBwdStride;
    static constexpr bool kReverse = true;       // planes back to front; each stage also carries the tile's saved transmittance
    static constexpr bool kSleepPolls = true;
    static constexpr bool kWideFact = false;     // the backward keeps the 56..88-wide classes: its shared memory is full
    static constexpr bool kBinaryCopies = false; // expanded MPI: one 4-row copy per lane (see staged_producer)
    // factored MPI: colour box = 3 copies of 12 rows (row offset r * 3 * bw * 4 bytes must be a multiple of 128 for bw = 56..88,
    // i.e. r a multiple of 4; 18-row halves gave cudaErrorMisalignedAddress)
    static constexpr int kColourCopyRows = 12;
    static_assert(kBwdMaxBH % kColourCopyRows == 0 && kColourCopyRows % 4 == 0, "colour copies tile the box, 128-byte aligned");
    // Magnification limit of the gradient box.  A fixed-point contribution is |c| 2^(kFixBits - e) < 2^25 w for alpha (2^21 w for
    // colour; w = the tap's bilinear weight, see tile_scale_exponent), plus 1/2 of rounding, and a tile has 64 x 24 = 1536 pixels:
    // a texel's int32 sum cannot wrap while the bilinear weights it collects from one tile add up to at most 63.  Over one tile a
    // pinhole camera maps pixels to texels at a nearly uniform scale of s texels per pixel, and one texel's weights summed along a
    // pixel row are at most 1/s + 1 (samples of a unit-area tent at spacing s); so the sum is at most (1/s + 1)^2 <= 49 when
    // s >= 1/kMagLimit.  The producer estimates s per (tile, plane) from the floored corner coordinates: a span of d texels over
    // ext pixels has s >= (d - 1) / ext.  It publishes a stage with kMagLimit (d - 1) < ext in either direction as not usable by
    // the fast body, which then takes the generic body (fp32 red.global.add, no limit).  The margin from 49 to 63 covers a rolled
    // camera (the corner box overstates s by up to 6 %) and the perspective change of s across a tile.  Magnifications beyond
    // about 6x (a 64^2 texture rendered at 512^2) pay for it; ray tensors that are not a pinhole camera's are judged by their
    // corner rays like any other footprint.
    static constexpr int kMagLimit = 6;
};

struct GradPairs {
    f2 g0[kPairs], g1[kPairs], g2[kPairs], gs[kPairs];   // upstream colour gradient and g_depth * (ray . z_dir)
};

// what the flushers need to know about a finished gradient box
struct __align__(16) GradMeta {
    int bx0, by0;        // texel coordinates of box element [0][.][0]
    int rows, cls;       // staged rows (0: nothing in the box), width class (bw = kMinBW + cls * kBWStep)
    int plane;           // m * N + i
    float scale;         // alpha channel: 2^(e_a - kFixBits), fixed point -> fp32
    int mpi_bg;          // factored MPI: 2 * m + (1 if this plane's colour gradient goes to g_bg_rgb: the last plane)
    float scale_rgb;     // colour channels: 2^(e_rgb - kFixBitsRgb)
};
constexpr int kBwdAlphaOff = 3 * kMaxBW * kBwdMaxBH;     // factored MPI: alpha box behind the colour box (floats / ints)

// red.global.add.f32 without a return value
__device__ __forceinline__ void red_add(float* p, float v) { asm volatile("red.global.add.f32 [%0], %1;" ::"l"(p), "f"(v) : "memory"); }
__device__ __forceinline__ void red_add_v4(float* p, float a, float b, float c, float d) {
    asm volatile("red.global.add.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(p), "f"(a), "f"(b), "f"(c), "f"(d) : "memory");
}

// Scatter one pixel's four channel gradients through its bilinear footprint straight into global memory
// (grid_sampler_2d_backward); the rare path of a warp whose footprints are not all inside the staged box.
// (The expanded instantiation passes one base pointer -- see sample_plane_direct for why -- the factored one four.)
__device__ __noinline__ void scatter_plane_global(float* __restrict__ gplane, size_t tex, int Wt, int Ht, int x0, int y0, float v0, float v1,
                                                  float v2, float v3, float w00, float w01, float w10, float w11) {
    const bool vx0 = (unsigned)x0 < (unsigned)Wt, vx1 = (unsigned)(x0 + 1) < (unsigned)Wt;
    const bool vy0 = (unsigned)y0 < (unsigned)Ht, vy1 = (unsigned)(y0 + 1) < (unsigned)Ht;
    float* b0 = gplane + ((long long)y0 * Wt + x0);
    const float v[4] = {v0, v1, v2, v3};
#pragma unroll
    for (int c = 0; c < 4; ++c, b0 += tex) {
        if (vx0 && vy0) red_add(b0, v[c] * w00);
        if (vx1 && vy0) red_add(b0 + 1, v[c] * w01);
        if (vx0 && vy1) red_add(b0 + Wt, v[c] * w10);
        if (vx1 && vy1) red_add(b0 + Wt + 1, v[c] * w11);
    }
}
__device__ __noinline__ void scatter_pixel_global(const GradChans gch, int Wt, int Ht, int x0, int y0, float v0, float v1,
                                                  float v2, float v3, float w00, float w01, float w10, float w11) {
    const bool vx0 = (unsigned)x0 < (unsigned)Wt, vx1 = (unsigned)(x0 + 1) < (unsigned)Wt;
    const bool vy0 = (unsigned)y0 < (unsigned)Ht, vy1 = (unsigned)(y0 + 1) < (unsigned)Ht;
    const long long o = (long long)y0 * Wt + x0;
    const float v[4] = {v0, v1, v2, v3};
#pragma unroll
    for (int c = 0; c < 4; ++c) {
        float* b0 = gch.c[c] + o;
        if (vx0 && vy0) red_add(b0, v[c] * w00);
        if (vx1 && vy0) red_add(b0 + 1, v[c] * w01);
        if (vx0 && vy1) red_add(b0 + Wt, v[c] * w10);
        if (vx1 && vy1) red_add(b0 + Wt + 1, v[c] * w11);
    }
}

// Fixed point.  Every contribution c of a tile satisfies |c| <= 2 qmax, where
// qmax = max over the tile's pixels of |G_r| + |G_g| + |G_b| + |G_d (ray . z_dir)| * max_i |scale_i|:
//   |dL/d rgb contribution| = |G_c| a T w <= qmax;   |dL/d a contribution| = T |q - R| w <= 2 qmax   (rgb, a, T, w in [0,1];
//   R is a sub-convex combination of the q's).  With 2^e > 4 qmax (a factor 2 of slack for inputs that leave [0,1] by rounding)
// contributions are rounded to multiples of 2^(e - kFixBits): |c| 2^(kFixBits - e) < 2^(kFixBits - 1), i.e. 25 bits + sign per
// contribution (finer than the fp32 accumulation it replaces whenever the running sum is within 4x of the bound), and a texel
// may collect 2^(31 - kFixBits + 1) = 64 contributions of maximum size in int32.  Magnified footprints, where one texel collects
// more than that from one tile, take the generic body (BwdRing::kMagLimit).
constexpr int kFixBits = 26, kFixSplit = 4;              // alpha: low kFixSplit bits come from the second conversion step
// The three colour channels have their own, tighter bound -- |dL/d rgb contribution| = |G_c| a T w <= gmax = max |G_c| over the
// tile, without the depth term and the factor 2 of the alpha bound -- and take the one-step conversion: 2^e_rgb > 2 gmax,
// contributions rounded to multiples of 2^(e_rgb - 22) (|c| 2^(22 - e_rgb) < 2^21: a factor 2 inside the 2^22 the magic constant
// allows, for inputs that leave [0,1] by rounding).
constexpr int kFixBitsRgb = 22;
constexpr float kMagicHi = 12582912.0f * 16.0f;          // 1.5 * 2^(23 + kFixSplit): ulp = 2^kFixSplit
constexpr int kMagicHiBits = 0x4b400000 + (kFixSplit << 23);
// Exponents for which 2^(kFixBits - e), 2^(e - kFixBits), 2^(kFixBitsRgb - e) and 2^(e - kFixBitsRgb) are all normal floats, so that
// scaling and flushing are exact: e >= -100 (2^(e - 26) >= 2^-126); every finite b gives e <= 128, and an infinite one 129.
// A tile whose exponents fall outside (an inf/NaN upstream gradient, |G| beyond about 1e37 or below about 1e-31) takes the
// generic body, which has no such limits.
constexpr int kMinScaleExp = -100, kMaxScaleExp = 128;
__device__ __forceinline__ int tile_scale_exponent(float qmax) {
    const float b = 4.0f * qmax;
    if (!(b > 0.0f)) return 0;
    return (int)((__float_as_uint(b) >> 23) & 0xffu) - 126;     // 2^e > b  (b = 1.m * 2^(E-127) < 2^(E-126))
}
// RN(x) for |x| < 2^(22 + kFixSplit), two pixels at once, as integers: the high part is read from the mantissa of x + 1.5 * 2^27
// (a multiple of 16), the exact remainder (|r| <= 8) from the mantissa of r + 1.5 * 2^23.  x = vF * w is never formed: both steps
// are FMAs on the exact product.
__device__ __forceinline__ void fix2(f2 vF, f2 w, int& ia, int& ib) {
    const f2 t1 = fma2(vF, w, splat(kMagicHi));
    const f2 nhi = fma2(t1, splat(-1.0f), splat(kMagicHi));      // -(high part), exact
    const f2 t2 = add2(fma2(vF, w, nhi), splat(kFloorMagic));    // remainder, rounded to an integer
    ia = ((__float_as_int(t1.x) - kMagicHiBits) << kFixSplit) + (__float_as_int(t2.x) - kFloorMagicBits);
    ib = ((__float_as_int(t1.y) - kMagicHiBits) << kFixSplit) + (__float_as_int(t2.y) - kFloorMagicBits);
}

// ---- deterministic backward (gmpi_mpi_render_bwd_deterministic_ex, DESIGN.md section 4.3) ----
// Every contribution becomes an integer in units of 2^(E - k), one E per call and channel kind (the box kernel's per-tile bound
// taken over all pixels of all views, mpi_bwd_det_bounds_kernel), and is added with red.global.add.u64 into int64 sums: integer
// addition is associative, so the sums do not depend on the order the hardware adds in.  An inf/NaN contribution sets a bit of
// its element instead (1 +inf, 2 -inf, 4 NaN; four bits per element).  mpi_bwd_det_finish_kernel turns both into fp32.
// The kernels address the sums through the gradient pointers of RenderParams, which point into the scratch viewed as floats:
// (dst - base) is the element index.
struct DetAcc {
    float* base;                 // scratch sums viewed as floats; the g_* pointers of the call's RenderParams point into it
    unsigned long long* acc;     // [G] int64 sums (two's complement)
    uint32_t* nf;                // [ceil(G / 8)] non-finite bits
    uint32_t* bounds;            // [2] bits of the call's qmax and gmax (non-negative floats)
    int k_a, k_rgb;              // fraction bits of the alpha and colour units (chosen per call on the host: no sum can wrap)
};
// The unit 2^ue of one channel kind and 2^-ue as the product of two normal floats (2^-ue itself can be out of float range).
struct DetUnit {
    float s0, s1;
    int ue;
};
// Clamp of the call's exponent: every scale constant of the box kernel is a normal float (as per tile)
__device__ __forceinline__ DetUnit det_unit(float bound, int k) {
    const int e = max(kMinScaleExp, min(kMaxScaleExp, tile_scale_exponent(bound)));
    const int sh = k - e, h = sh / 2;
    DetUnit u;
    u.s0 = __uint_as_float((unsigned)(127 + h) << 23);
    u.s1 = __uint_as_float((unsigned)(127 + sh - h) << 23);
    u.ue = e - k;
    return u;
}
__device__ __forceinline__ void det_add_int(const DetAcc& d, size_t i, long long x) {
    if (x) asm volatile("red.global.add.u64 [%0], %1;" ::"l"(d.acc + i), "l"(x) : "memory");
}
// one fp32 contribution c to the element `dst` points at (a pointer into DetAcc::base)
__device__ __forceinline__ void det_add(const DetAcc& d, const DetUnit& u, const float* dst, float c) {
    const size_t i = (size_t)(dst - d.base);
    if (!(fabsf(c) <= 0x1.fffffep127f)) {
        const uint32_t bit = c != c ? 4u : c > 0.0f ? 1u : 2u;
        atomicOr(d.nf + (i >> 3), bit << ((i & 7) * 4));
        return;
    }
    det_add_int(d, i, __float2ll_rn(__fmul_rn(__fmul_rn(c, u.s0), u.s1)));     // exact scaling, one rounding to the unit
}
// A tile's fixed-point sum s in units 2^te -> units 2^ue: exact when te >= ue, else rounded to nearest, ties away from zero.
// (|s 2^(te - ue)| < 2^62 by the choice of k: the shift cannot overflow.)
__device__ __forceinline__ long long det_rescale(int s, int te, int ue) {
    const int sh = te - ue;
    if (sh >= 0) return (long long)((unsigned long long)(long long)s << sh);
    if (sh < -31) return 0;                                   // |s| <= 2^31: |s| 2^sh < 1/2
    const long long a = s < 0 ? -(long long)s : (long long)s;
    const long long q = (a + (1ll << (-sh - 1))) >> -sh;
    return s < 0 ? -q : q;
}

// The call's scale pre-pass and the finish pass of the deterministic backward.
// bounds[0] = max over every pixel of every view of the box kernel's per-pixel alpha bound |G_r| + |G_g| + |G_b| + |G_d dz| *
// max_i |z_diff_i| / |ray_z| (the same float operations as the tile bound of bwd_box_body, so no tile's exponent exceeds the
// call's); bounds[1] = max |G_c|.  Pixels with an inf/NaN upstream gradient are left out of bounds[0] and non-finite
// components out of bounds[1]: their contributions go to the non-finite bits.  Integer atomicMax on the bits of non-negative
// floats: independent of order.  Grid (pixel blocks, min(V, 65535)) of 256 threads; block row y takes views y, y + gridDim.y, ...
__global__ void __launch_bounds__(256)
mpi_bwd_det_bounds_kernel(const RenderParams p, uint32_t* __restrict__ bounds) {
    __shared__ unsigned s_zmax;
    const size_t img = (size_t)p.H * p.W, pix = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    const float gscale = (p.options & GMPI_COLOR_MINUS1_1) ? 2.0f : 1.0f;
    float qmax = 0.0f, gmax = 0.0f;
    for (int v = blockIdx.y; v < p.V; v += gridDim.y) {
        const int m = __ldg(p.view2mpi + v);
        const float ev[3] = {__ldg(p.eye + 3 * v), __ldg(p.eye + 3 * v + 1), __ldg(p.eye + 3 * v + 2)};
        const float zd[3] = {__ldg(p.z_dir + 3 * v), __ldg(p.z_dir + 3 * v + 1), __ldg(p.z_dir + 3 * v + 2)};
        __syncthreads();
        if (threadIdx.x == 0) s_zmax = 0u;
        __syncthreads();
        float zm = 0.0f;
        for (int i = threadIdx.x; i < p.N; i += blockDim.x)
            zm = fmaxf(zm, fabsf(make_plane_const(p.dhw + ((size_t)m * p.N + i) * 3, ev[2]).z_diff));
        atomicMax(&s_zmax, __float_as_uint(zm));
        __syncthreads();
        const float zmax = __uint_as_float(s_zmax);
        if (pix < img) {
            const float* rd = p.ray_dir + (size_t)v * 3 * img + pix;
            const RayConst rc = make_ray_const(__ldg(rd), __ldg(rd + img), __ldg(rd + 2 * img), ev, zd);
            const float* gc = p.g_color + (size_t)v * 3 * img + pix;
            const float g0 = gscale * __ldg(gc), g1 = gscale * __ldg(gc + img), g2 = gscale * __ldg(gc + 2 * img);
            const float g3 = p.g_depth ? __ldg(p.g_depth + (size_t)v * img + pix) * rc.dz : 0.0f;
            const float ga = fabsf(g0) + fabsf(g1) + fabsf(g2), gd = fabsf(g3);
            if (ga + gd <= 0x1.fffffep127f) qmax = fmaxf(qmax, ga + gd * (zmax * fabsf(rc.yrz)));   // NaN (0 * inf) is dropped
            const auto fin = [](float x) { return fabsf(x) <= 0x1.fffffep127f ? fabsf(x) : 0.0f; };
            gmax = fmaxf(gmax, fmaxf(fin(g0), fmaxf(fin(g1), fin(g2))));
        }
    }
    for (int o = 16; o > 0; o >>= 1) {
        qmax = fmaxf(qmax, __shfl_xor_sync(0xffffffffu, qmax, o));
        gmax = fmaxf(gmax, __shfl_xor_sync(0xffffffffu, gmax, o));
    }
    if ((threadIdx.x & 31) == 0) {
        if (qmax > 0.0f) atomicMax(bounds, __float_as_uint(qmax));
        if (gmax > 0.0f) atomicMax(bounds + 1, __float_as_uint(gmax));
    }
}

// The finish pass: element i of the sums (layout: g_rgba, or g_rgb | g_alpha | g_bg_rgb) -> fp32, written (`zero`) or added into
// the caller's gradient.  Non-finite bits give what an fp32 sum of the contributions gives: NaN if a NaN or both infinities were
// added, else the infinity.  seg1 / seg2: first elements of g_alpha and g_bg_rgb in the sums (factored; G otherwise).
__global__ void __launch_bounds__(256)
mpi_bwd_det_finish_kernel(const DetAcc da, float* __restrict__ g0, float* __restrict__ g1, float* __restrict__ g2, size_t G, size_t seg1,
                          size_t seg2, size_t tex, bool factored, bool zero) {
    const DetUnit ua = det_unit(__uint_as_float(__ldg(da.bounds)), da.k_a);
    const DetUnit urgb = det_unit(0.5f * __uint_as_float(__ldg(da.bounds + 1)), da.k_rgb);
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < G; i += (size_t)gridDim.x * blockDim.x) {
        const bool alpha = factored ? (i >= seg1 && i < seg2) : (i / tex) % 4 == 3;
        const uint32_t nf = (__ldcs(da.nf + (i >> 3)) >> ((i & 7) * 4)) & 7u;
        float x;
        if (nf) {
            x = (nf & 4u) || nf == 3u ? __int_as_float(0x7fffffff) : nf == 1u ? INFINITY : -INFINITY;
        } else {
            // RN to fp32, then an exact power-of-two scale in two normal steps (a result below the normal range rounds once more)
            const int ue = alpha ? ua.ue : urgb.ue, h = ue / 2;
            x = __ll2float_rn((long long)__ldcs(da.acc + i));
            x = __fmul_rn(__fmul_rn(x, __uint_as_float((unsigned)(127 + h) << 23)), __uint_as_float((unsigned)(127 + ue - h) << 23));
        }
        float* dst = i < seg1 ? g0 + i : i < seg2 ? g1 + (i - seg1) : g2 + (i - seg2);
        *dst = zero ? x : *dst + x;
    }
}

__device__ __noinline__ void scatter_plane_det(const DetAcc& da, const DetUnit& ua, const DetUnit& urgb, float* __restrict__ gplane,
                                               size_t tex, int Wt, int Ht, int x0, int y0, float v0, float v1, float v2, float v3,
                                               float w00, float w01, float w10, float w11) {
    const bool vx0 = (unsigned)x0 < (unsigned)Wt, vx1 = (unsigned)(x0 + 1) < (unsigned)Wt;
    const bool vy0 = (unsigned)y0 < (unsigned)Ht, vy1 = (unsigned)(y0 + 1) < (unsigned)Ht;
    float* b0 = gplane + ((long long)y0 * Wt + x0);
    const float v[4] = {v0, v1, v2, v3};
#pragma unroll
    for (int c = 0; c < 4; ++c, b0 += tex) {
        const DetUnit& u = c == 3 ? ua : urgb;
        if (vx0 && vy0) det_add(da, u, b0, v[c] * w00);
        if (vx1 && vy0) det_add(da, u, b0 + 1, v[c] * w01);
        if (vx0 && vy1) det_add(da, u, b0 + Wt, v[c] * w10);
        if (vx1 && vy1) det_add(da, u, b0 + Wt + 1, v[c] * w11);
    }
}
__device__ __noinline__ void scatter_pixel_det(const DetAcc& da, const DetUnit& ua, const DetUnit& urgb, const GradChans gch, int Wt,
                                               int Ht, int x0, int y0, float v0, float v1, float v2, float v3, float w00, float w01,
                                               float w10, float w11) {
    const bool vx0 = (unsigned)x0 < (unsigned)Wt, vx1 = (unsigned)(x0 + 1) < (unsigned)Wt;
    const bool vy0 = (unsigned)y0 < (unsigned)Ht, vy1 = (unsigned)(y0 + 1) < (unsigned)Ht;
    const long long o = (long long)y0 * Wt + x0;
    const float v[4] = {v0, v1, v2, v3};
#pragma unroll
    for (int c = 0; c < 4; ++c) {
        const DetUnit& u = c == 3 ? ua : urgb;
        float* b0 = gch.c[c] + o;
        if (vx0 && vy0) det_add(da, u, b0, v[c] * w00);
        if (vx1 && vy0) det_add(da, u, b0 + 1, v[c] * w01);
        if (vx0 && vy1) det_add(da, u, b0 + Wt, v[c] * w10);
        if (vx1 && vy1) det_add(da, u, b0 + Wt + 1, v[c] * w11);
    }
}

// One (pair, channel) of the scatter: the four bilinear contributions of two pixels into the gradient box.
template <int PITCH, bool kTwoStep>
__device__ __forceinline__ void scatter_channel(int* __restrict__ ga, int* __restrict__ gq, f2 vF, const f2 (&w)[4]) {
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        int ca, cb;
        if (!kTwoStep) {     // RN(vF * w) read from the mantissa of one packed FMA
            const f2 t = fma2(vF, w[k], splat(kFloorMagic));
            ca = __float_as_int(t.x) - kFloorMagicBits; cb = __float_as_int(t.y) - kFloorMagicBits;
        } else {
            fix2(vF, w[k], ca, cb);
        }
        const int off = (k & 1) + (k >> 1) * PITCH;
        atomicAdd(ga + off, ca);
        atomicAdd(gq + off, cb);
    }
}

// Fast body: four pixels (two packed pairs) from a staged box of compile-time width BW: sample, form the gradients, add the 64
// fixed-point contributions to the gradient box `gb` (same layout as the staged box).  Returns false (nothing sampled, R
// unchanged, nothing added) if any footprint is not inside the box.
// AOFF as in BoxTaps: 0 = expanded stage, > 0 = factored (colour box [row][3][BW], alpha box [row][BW] at AOFF).
// Each pair is scattered as soon as it is formed: keeping both pairs' weights and values alive until a later scatter phase costs
// ~36 registers and spills.
template <int BW, int AOFF = 0>
__device__ __forceinline__ bool bwd_box_pairs(const float* __restrict__ sb, int* __restrict__ gb, int cx, int cy, int rows2, const CoordPairs& c,
                                              const f2 (&T)[kPairs], const GradPairs& G, f2 (&R)[kPairs], f2 Fs, f2 Fs_rgb,
                                              uint64_t* g_empty_bar, uint32_t g_empty_parity) {
    using Box = BoxTaps<BW, AOFF>;
    const f2 m1 = splat(-1.0f);
    Box bt;
    if (!bt.locate(cx, cy, rows2, c)) return false;
#pragma unroll
    for (int P = 0; P < kPairs; ++P) {
        f2 w[4], r, g, b, a;
        bt.sample(sb, c, P, w, r, g, b, a);
        const f2 q = fma2(G.g0[P], r, fma2(G.g1[P], g, fma2(G.g2[P], b, mul2(G.gs[P], c.sc[P]))));
        const f2 d = fma2(R[P], m1, q);                 // q - R
        const f2 wT = mul2(a, T[P]);
        R[P] = fma2(a, d, R[P]);
        // ---- scatter (grid_sampler_2d_backward), fixed point: colour channels one-step, alpha two-step ----
        // The gradient box is needed only from here on: the flushers get the first pair's sampling time to finish emptying it.
        if (P == 0) mbar_wait(g_empty_bar, g_empty_parity);
        const f2 wF = mul2(wT, Fs_rgb);                 // exact (power of two)
        int* ga = gb + bt.ia[P];
        int* gq = gb + bt.ib[P];
        scatter_channel<Box::RP, false>(ga, gq, mul2(G.g0[P], wF), w);
        scatter_channel<Box::RP, false>(ga + BW, gq + BW, mul2(G.g1[P], wF), w);
        scatter_channel<Box::RP, false>(ga + 2 * BW, gq + 2 * BW, mul2(G.g2[P], wF), w);
        scatter_channel<Box::AP, true>(AOFF ? gb + bt.ja[P] : ga + Box::A0, AOFF ? gb + bt.jb[P] : gq + Box::A0, mul2(mul2(T[P], d), Fs), w);   // dL/d alpha
    }
    return true;
}

// Flusher: rows fw, fw + 3, ... of a finished gradient box -> fp32 -> red.global.add.v4.f32, then zero.
// kDet: the box's integer sums go to the deterministic sums instead, converted to the call's units (ue_a, ue_rgb).
template <int BW, bool FAC, bool kDet = false>
__device__ __forceinline__ void flush_box(int* __restrict__ gb, const GradMeta& gm, const RenderParams& p, size_t tex, int Ht, int Wt,
                                          int fw, int lane, const DetAcc& da, int ue_a, int ue_rgb) {
    constexpr int Q = BW / 4;      // float4 quads per channel row
    // destination slabs of the four channels
    float* dst[4];
    if (FAC) {
        float* rgb = ((gm.mpi_bg & 1) ? p.g_bg_rgb : p.g_rgb) + (size_t)(gm.mpi_bg >> 1) * 3 * tex;
        dst[0] = rgb; dst[1] = rgb + tex; dst[2] = rgb + 2 * tex; dst[3] = p.g_alpha + (size_t)gm.plane * tex;
    } else {
        float* b = p.g_rgba + (size_t)gm.plane * 4 * tex;
        dst[0] = b; dst[1] = b + tex; dst[2] = b + 2 * tex; dst[3] = b + 3 * tex;
    }
    constexpr int kRowsPerWarp = (kBwdMaxBH + kBwdFlushWarps - 1) / kBwdFlushWarps;
    // BW quads per box row: channel ch, quad x4.  Expanded: [row][4][BW]; factored: [row][3][BW] + alpha box [row][BW].
    // All rows of this warp are loaded before any is processed: the flush is a latency chain otherwise (LDS -> test -> RED).
    for (int j = lane; j < BW; j += 32) {
        const int ch = j / Q, x4 = j - ch * Q;
        const int cell0 = FAC ? (ch < 3 ? j * 4 : kBwdAlphaOff + x4 * 4) : j * 4;          // int offset inside a row
        constexpr int kColPitch = FAC ? 3 * BW : 4 * BW;
        const int pitch = (FAC && ch == 3) ? BW : kColPitch;
        int4 a[kRowsPerWarp];
#pragma unroll
        for (int k = 0; k < kRowsPerWarp; ++k) {
            const int r = fw + k * kBwdFlushWarps;
            a[k] = *reinterpret_cast<const int4*>(gb + r * pitch + cell0);      // rows beyond gm.rows are never written: they read 0
        }
        const int tx = gm.bx0 + 4 * x4;
        const bool col_ok = (unsigned)tx < (unsigned)Wt;          // bx0 % 4 == 0 and Wt % 4 == 0: a quad is inside or outside as a whole
        float* d = (ch == 0 ? dst[0] : ch == 1 ? dst[1] : ch == 2 ? dst[2] : dst[3]) + tx;
        const float sc = ch < 3 ? gm.scale_rgb : gm.scale;
#pragma unroll
        for (int k = 0; k < kRowsPerWarp; ++k) {
            const int r = fw + k * kBwdFlushWarps;
            if ((a[k].x | a[k].y | a[k].z | a[k].w) == 0) continue;  // untouched halo (or a row beyond the box): nothing to add or clear
            *reinterpret_cast<int4*>(gb + r * pitch + cell0) = make_int4(0, 0, 0, 0);
            const int ty = gm.by0 + r;
            if constexpr (kDet) {
                if (col_ok && (unsigned)ty < (unsigned)Ht) {
                    const int te = (int)((__float_as_uint(sc) >> 23) & 0xffu) - 127, ue = ch < 3 ? ue_rgb : ue_a;   // sc = 2^te
                    const size_t i = (size_t)(d + (size_t)ty * Wt - da.base);
                    det_add_int(da, i, det_rescale(a[k].x, te, ue));
                    det_add_int(da, i + 1, det_rescale(a[k].y, te, ue));
                    det_add_int(da, i + 2, det_rescale(a[k].z, te, ue));
                    det_add_int(da, i + 3, det_rescale(a[k].w, te, ue));
                }
            } else if (col_ok && (unsigned)ty < (unsigned)Ht)
                red_add_v4(d + (size_t)ty * Wt, (float)a[k].x * sc, (float)a[k].y * sc, (float)a[k].z * sc, (float)a[k].w * sc);
        }
    }
}

// The box kernel's body; kDet: the deterministic instantiation (flush and generic-body scatter into DetAcc `da`).
template <bool kAlignCorners, bool kFactored, bool kDet>
__device__ __forceinline__ void bwd_box_body(const RenderParams p, const TmaMaps& maps, const int tiles_x, const int tiles_y,
                                             const DetAcc da) {
    extern __shared__ __align__(1024) unsigned char smem_raw[];
    float* s_buf = reinterpret_cast<float*>(smem_raw);                                          // rgba ring (+ transmittance boxes)
    int* s_grad = reinterpret_cast<int*>(smem_raw + (size_t)kBwdStages * kBwdStride * 4);       // gradient boxes
    PlaneConst* s_pc = reinterpret_cast<PlaneConst*>(smem_raw + (size_t)(kBwdStages * kBwdStride + kBwdBoxes * kBwdPlaneFloats) * 4);
    __shared__ StageMeta s_meta[kBwdStages];
    __shared__ GradMeta s_gmeta[kBwdBoxes];
    __shared__ __align__(8) uint64_t s_full[kBwdStages], s_empty[kBwdStages], g_full[kBwdBoxes], g_empty[kBwdBoxes];
    __shared__ TileWalk s_walk;
    __shared__ unsigned s_qmax[3], s_gmax[3];   // per-tile bounds (bits of non-negative floats), three slots in rotation
    __shared__ unsigned s_zmax;           // max_i |z_diff_i| of the current view's plane table

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    if (threadIdx.x == 0) {
        s_walk.init(tiles_x, p.H, p.V, (int)blockIdx.x, (int)gridDim.x, kBwdTileH, p.view_group);
        for (int s = 0; s < kBwdStages; ++s) {
            mbar_init(&s_full[s], 1);
            mbar_init(&s_empty[s], kBwdConsWarps);
        }
        for (int s = 0; s < kBwdBoxes; ++s) {
            mbar_init(&g_full[s], kBwdConsWarps);
            mbar_init(&g_empty[s], kBwdFlushWarps);
        }
        s_qmax[0] = s_qmax[1] = s_qmax[2] = 0u;
        s_gmax[0] = s_gmax[1] = s_gmax[2] = 0u;
        s_zmax = 0u;
        fence_mbar_init();
    }
    for (int i = threadIdx.x; i < kBwdBoxes * kBwdPlaneFloats; i += kBwdThreads) s_grad[i] = 0;
    __syncthreads();

    const int Ht = p.Ht, Wt = p.Wt, N = p.N;
    const size_t tex = (size_t)Ht * Wt;

    if (warp == kBwdConsWarps) {
        // ================================ producer ================================
        if (lane == 0) tma_prefetch_desc(&maps.t);
        staged_producer<kAlignCorners, BwdRing, kFactored>(p, maps, s_buf, s_meta, s_full, s_empty, &s_walk, lane);
    } else if (warp > kBwdConsWarps) {
        // ================================ flushers ================================
        const int fw = warp - kBwdConsWarps - 1;
        int ue_a = 0, ue_rgb = 0;
        if constexpr (kDet) {
            ue_a = det_unit(__uint_as_float(__ldg(da.bounds)), da.k_a).ue;
            ue_rgb = det_unit(0.5f * __uint_as_float(__ldg(da.bounds + 1)), da.k_rgb).ue;
        }
        int f_box = 0;
        uint32_t f_phase = 0;
        TileXY txy;
        for (int j = 0; s_walk.at(j, txy); ++j) {
            for (int ii = 0; ii < N; ++ii) {
                const int b = f_box;
                const uint32_t ph = f_phase;
                if (++f_box == kBwdBoxes) { f_box = 0; f_phase ^= 1u; }
                mbar_wait_sleep(&g_full[b], ph);
                const GradMeta gm = s_gmeta[b];
                int* gb = s_grad + b * kBwdPlaneFloats;
                if (gm.rows > 0) {
                    switch (gm.cls) {     // warp-uniform
                        case 0: flush_box<56, kFactored, kDet>(gb, gm, p, tex, Ht, Wt, fw, lane, da, ue_a, ue_rgb); break;
                        case 1: flush_box<64, kFactored, kDet>(gb, gm, p, tex, Ht, Wt, fw, lane, da, ue_a, ue_rgb); break;
                        case 2: flush_box<72, kFactored, kDet>(gb, gm, p, tex, Ht, Wt, fw, lane, da, ue_a, ue_rgb); break;
                        case 3: flush_box<80, kFactored, kDet>(gb, gm, p, tex, Ht, Wt, fw, lane, da, ue_a, ue_rgb); break;
                        default: flush_box<88, kFactored, kDet>(gb, gm, p, tex, Ht, Wt, fw, lane, da, ue_a, ue_rgb); break;
                    }
                }
                __syncwarp();
                mbar_arrive_if(&g_empty[b], lane == 0);
            }
        }
    } else {
        // ================================ consumers ================================
        const float fWt = (float)Wt, fHt = (float)Ht;
        float hsx = 0.5f * (float)(Wt - 1), hsy = 0.5f * (float)(Ht - 1);
        int lane_ = lane;
        asm volatile("" : "+f"(hsx), "+f"(hsy), "+r"(lane_));     // opaque: not re-derived from the parameters in every plane iteration
        const size_t img = (size_t)p.H * p.W;
        int c_stage = 0, g_box = 0;
        uint32_t c_phase = 0, g_phase = 0;
        const float gscale = (p.options & GMPI_COLOR_MINUS1_1) ? 2.0f : 1.0f;   // upstream gradient is w.r.t. 2*color-1
        int v_table = -1;
        TileXY txy;
        for (int j = 0; s_walk.at(j, txy); ++j) {
            const int v = txy.v, px0 = txy.px0, py0 = txy.py0;
            const int m = __ldg(p.view2mpi + v);
            const float* e = p.eye + 3 * v;
            const float ev[3] = {__ldg(e), __ldg(e + 1), __ldg(e + 2)};
            const float zd[3] = {__ldg(p.z_dir + 3 * v), __ldg(p.z_dir + 3 * v + 1), __ldg(p.z_dir + 3 * v + 2)};
            if (v != v_table) {          // (view, plane) constants, once per view and CTA
                consumer_bar_sync<kBwdConsThreads>();
                if (threadIdx.x == 0) s_zmax = 0u;
                consumer_bar_sync<kBwdConsThreads>();
                float zm = 0.0f;
                for (int i = threadIdx.x; i < N; i += kBwdConsThreads) {
                    const PlaneConst pc = make_plane_const(p.dhw + ((size_t)m * N + i) * 3, ev[2]);
                    s_pc[i] = pc;
                    zm = fmaxf(zm, fabsf(pc.z_diff));
                }
                atomicMax(&s_zmax, __float_as_uint(zm));
                consumer_bar_sync<kBwdConsThreads>();
                v_table = v;
            }
            // ---- per-pixel inputs (clamped into the image; the tile overhang carries zero upstream gradient) ----
            const float* rays = p.ray_dir + (size_t)v * 3 * img;
            RayConst rc[kPix];
            RayPairs rp;
            GradPairs G;
            float gq[kPix][4];
            bool rays_fast = (in_safe_range(ev[0]) || ev[0] == 0.0f) && (in_safe_range(ev[1]) || ev[1] == 0.0f);
            const float zmax = __uint_as_float(s_zmax);
            float qmax = 0.0f, gmax = 0.0f;
#pragma unroll
            for (int q = 0; q < kPix; ++q) {
                const int pxq = px0 + lane + 32 * (q & 1), pyq = py0 + kPairs * warp + (q >> 1);
                const bool valid = pxq < p.W && pyq < p.H;
                const size_t pix = (size_t)min(pyq, p.H - 1) * p.W + min(pxq, p.W - 1);
                const float* rd = rays + pix;
                rc[q] = make_ray_const(__ldg(rd), __ldg(rd + img), __ldg(rd + 2 * img), ev, zd);
                rays_fast = rays_fast && rc[q].fast && fabsf(rc[q].rx2) <= 0x1p40f && fabsf(rc[q].ry2) <= 0x1p40f;
                const float* gc = p.g_color + (size_t)v * 3 * img + pix;
                gq[q][0] = valid ? gscale * __ldg(gc) : 0.0f;
                gq[q][1] = valid ? gscale * __ldg(gc + img) : 0.0f;
                gq[q][2] = valid ? gscale * __ldg(gc + 2 * img) : 0.0f;
                gq[q][3] = (valid && p.g_depth) ? __ldg(p.g_depth + (size_t)v * img + pix) * rc[q].dz : 0.0f;
                const float ga = fabsf(gq[q][0]) + fabsf(gq[q][1]) + fabsf(gq[q][2]), gd = fabsf(gq[q][3]);
                qmax = fmaxf(qmax, ga + gd * (zmax * fabsf(rc[q].yrz)));
                if (!(ga + gd <= 0x1.fffffep127f)) qmax = INFINITY;     // inf/NaN upstream gradient (fmaxf would drop a NaN)
                gmax = fmaxf(gmax, fmaxf(fabsf(gq[q][0]), fmaxf(fabsf(gq[q][1]), fabsf(gq[q][2]))));
            }
            // ---- the tile's fixed-point scale: max over all consumer threads (three slots in rotation, see below) ----
            {
                const int slot = j % 3;
                for (int o = 16; o > 0; o >>= 1) {
                    qmax = fmaxf(qmax, __shfl_xor_sync(0xffffffffu, qmax, o));
                    gmax = fmaxf(gmax, __shfl_xor_sync(0xffffffffu, gmax, o));
                }
                if (lane == 0) { atomicMax(&s_qmax[slot], __float_as_uint(qmax)); atomicMax(&s_gmax[slot], __float_as_uint(gmax)); }
                if (threadIdx.x == 0) s_qmax[(j + 1) % 3] = s_gmax[(j + 1) % 3] = 0u;   // next tile's slots: their last readers passed the previous tile's barrier
                consumer_bar_sync<kBwdConsThreads>();
                qmax = __uint_as_float(s_qmax[slot]);
                gmax = __uint_as_float(s_gmax[slot]);
            }
            int e_fix = tile_scale_exponent(qmax);
            int e_rgb = tile_scale_exponent(0.5f * gmax);                                         // 2^e_rgb > 2 gmax
            // CTA-uniform: the bounds are reduced over the tile.  Out of range, the tile takes the generic body (and the clamp
            // only keeps the unused constants well-formed)
            const bool scale_ok = e_fix >= kMinScaleExp && e_fix <= kMaxScaleExp && e_rgb >= kMinScaleExp && e_rgb <= kMaxScaleExp;
            e_fix = max(kMinScaleExp, min(kMaxScaleExp, e_fix));
            e_rgb = max(kMinScaleExp, min(kMaxScaleExp, e_rgb));
            const f2 Fs = splat(__uint_as_float((unsigned)(127 + kFixBits - e_fix) << 23));      // 2^(kFixBits - e)
            const float inv_scale = __uint_as_float((unsigned)(127 - kFixBits + e_fix) << 23);    // 2^(e - kFixBits)
            const f2 Fs_rgb = splat(__uint_as_float((unsigned)(127 + kFixBitsRgb - e_rgb) << 23));
            const float inv_scale_rgb = __uint_as_float((unsigned)(127 - kFixBitsRgb + e_rgb) << 23);

            const bool idle = py0 + kPairs * warp >= p.H;      // warp-uniform: no row of this warp is inside the image
            pack_ray_pairs(rc, rp);
#pragma unroll
            for (int P = 0; P < kPairs; ++P) {
                G.g0[P] = make_float2(gq[2 * P][0], gq[2 * P + 1][0]);
                G.g1[P] = make_float2(gq[2 * P][1], gq[2 * P + 1][1]);
                G.g2[P] = make_float2(gq[2 * P][2], gq[2 * P + 1][2]);
                G.gs[P] = make_float2(gq[2 * P][3], gq[2 * P + 1][3]);
            }
            const f2 ex2 = splat(rc[0].ex2), ey2 = splat(rc[0].ey2), hsx2 = splat(hsx), hsy2 = splat(hsy);
            const bool warp_fast = __all_sync(0xffffffffu, rays_fast) && !idle && scale_ok;
            f2 R[kPairs];
#pragma unroll
            for (int P = 0; P < kPairs; ++P) R[P] = splat(0.0f);
            for (int ii = 0; ii < N; ++ii) {
                const int i = N - 1 - ii;
                const int s = c_stage, b = g_box;
                const uint32_t ph = c_phase, gph = g_phase;
                if (++c_stage == kBwdStages) { c_stage = 0; c_phase ^= 1u; }
                if (++g_box == kBwdBoxes) { g_box = 0; g_phase ^= 1u; }
                const PlaneConst pcc = s_pc[i];
                CoordPairs cc;
                if (warp_fast) coords_pairs<kAlignCorners>(pcc, rp, ex2, ey2, hsx2, hsy2, fWt, fHt, cc);
                mbar_wait(&s_full[s], ph);
                const StageMeta mt = s_meta[s];
                const float* sb = s_buf + s * kBwdStride;
                const int sel = mt.sel;
                f2 T[kPairs];      // transmittance saved by the forward, staged next to the plane tile: [kBwdTileH][kTileW]
#pragma unroll
                for (int P = 0; P < kPairs; ++P) {
                    const float* tr = sb + kBwdPlaneFloats + (kPairs * warp + P) * kTileW + lane;
                    T[P] = make_float2(tr[0], tr[32]);
                }
                // ---- gradient box of this (tile, plane): sample, wait until the flushers have emptied it, scatter ----
                int* gb = s_grad + b * kBwdPlaneFloats;
                constexpr int AO = kFactored ? kBwdAlphaOff : 0;
                bool done = false;
                if (warp_fast) {   // warp-uniform, one-hot class
                    if (sel & (1 << 18)) done = bwd_box_pairs<72, AO>(sb, gb, mt.cx, mt.cy, mt.rows2, cc, T, G, R, Fs, Fs_rgb, &g_empty[b], gph ^ 1u);
                    else if (sel & (1 << 17)) done = bwd_box_pairs<64, AO>(sb, gb, mt.cx, mt.cy, mt.rows2, cc, T, G, R, Fs, Fs_rgb, &g_empty[b], gph ^ 1u);
                    else if (sel & (1 << 19)) done = bwd_box_pairs<80, AO>(sb, gb, mt.cx, mt.cy, mt.rows2, cc, T, G, R, Fs, Fs_rgb, &g_empty[b], gph ^ 1u);
                    else if (sel & (1 << 16)) done = bwd_box_pairs<56, AO>(sb, gb, mt.cx, mt.cy, mt.rows2, cc, T, G, R, Fs, Fs_rgb, &g_empty[b], gph ^ 1u);
                    else if (sel & (1 << 20)) done = bwd_box_pairs<88, AO>(sb, gb, mt.cx, mt.cy, mt.rows2, cc, T, G, R, Fs, Fs_rgb, &g_empty[b], gph ^ 1u);
                }
                const int cls = done ? 0 : -1;
                // a warp that did not use the box still waits: it must not arrive on g_full[b] a second time before the flushers
                // have taken the previous fill (the arrival counts of two fills would mix)
                if (!done) mbar_wait(&g_empty[b], gph ^ 1u);
                __syncwarp();
                mbar_arrive_if(&s_empty[s], lane_ == 0);    // taps and transmittance are consumed: hand the stage back
                if (warp == 0 && lane == 0) {               // (warp 0 always has a row inside the image)
                    GradMeta gm;
                    const int mode = (sel >> 8) & 3;
                    gm.bx0 = mt.cx - kFloorMagicBits; gm.by0 = mt.cy - kFloorMagicBits;
                    gm.rows = mode == 0 ? mt.rows2 + 2 : 0;
                    gm.cls = ((sel & 0xff) - kMinBW) / kBWStep;
                    gm.plane = m * N + i;
                    gm.scale = inv_scale;
                    gm.scale_rgb = inv_scale_rgb;
                    gm.mpi_bg = 2 * m + ((kFactored && p.g_bg_rgb && i == N - 1) ? 1 : 0);
                    s_gmeta[b] = gm;
                }
                __syncwarp();
                mbar_arrive_if(&g_full[b], lane_ == 0);
                if (cls < 0 && !idle) {
                    // ---- generic body (rare): per-pixel checks, sampling and scattering straight in global memory.  Also
                    // taken when the producer's corner-ray estimate says "nothing under the tile": a hint, never trusted ----
                    const float* plane = kFactored ? nullptr : p.rgba + ((size_t)m * N + i) * 4 * tex;
                    float* gplane = kFactored ? nullptr : p.g_rgba + ((size_t)m * N + i) * 4 * tex;
                    float* Rs = reinterpret_cast<float*>(R);
                    const float* Ts = reinterpret_cast<const float*>(T);
                    DetUnit ua{}, urgb{};
                    if constexpr (kDet) {
                        ua = det_unit(__uint_as_float(__ldg(da.bounds)), da.k_a);
                        urgb = det_unit(0.5f * __uint_as_float(__ldg(da.bounds + 1)), da.k_rgb);
                    }
#pragma unroll
                    for (int q = 0; q < kPix; ++q) {
                        const int qq = (q & 1) + 2 * (q >> 1);      // R / T are stored as pairs: element (P, half) = 2 P + half
                        RayConst rg = rc[q];
                        rg.fast = false;
                        const TexCoord tc = plane_coord<kAlignCorners>(pcc, rg, hsx, hsy, fWt, fHt);
                        if (!coord_hits(tc.ix, tc.iy, fWt, fHt)) continue;
                        const float4 sv = sample_plane_any<kFactored>(p, plane, m, i, tex, tc.ix, tc.iy);
                        const float fx = floorf(tc.ix), fy = floorf(tc.iy);
                        const float wx1 = tc.ix - fx, wy1 = tc.iy - fy, wx0 = 1.0f - wx1, wy0 = 1.0f - wy1;
                        const float qv = fmaf(gq[q][0], sv.x, fmaf(gq[q][1], sv.y, fmaf(gq[q][2], sv.z, gq[q][3] * tc.scale)));
                        const float d = qv - Rs[qq];
                        const float w = sv.w * Ts[qq];
                        Rs[qq] = fmaf(sv.w, d, Rs[qq]);
                        if constexpr (kDet) {
                            if (kFactored)
                                scatter_pixel_det(da, ua, urgb, grad_chans(p, m, i, tex), Wt, Ht, (int)fx, (int)fy, gq[q][0] * w,
                                                  gq[q][1] * w, gq[q][2] * w, Ts[qq] * d, wx0 * wy0, wx1 * wy0, wx0 * wy1, wx1 * wy1);
                            else
                                scatter_plane_det(da, ua, urgb, gplane, tex, Wt, Ht, (int)fx, (int)fy, gq[q][0] * w, gq[q][1] * w,
                                                  gq[q][2] * w, Ts[qq] * d, wx0 * wy0, wx1 * wy0, wx0 * wy1, wx1 * wy1);
                        } else if (kFactored)
                            scatter_pixel_global(grad_chans(p, m, i, tex), Wt, Ht, (int)fx, (int)fy, gq[q][0] * w, gq[q][1] * w, gq[q][2] * w,
                                                 Ts[qq] * d, wx0 * wy0, wx1 * wy0, wx0 * wy1, wx1 * wy1);
                        else
                            scatter_plane_global(gplane, tex, Wt, Ht, (int)fx, (int)fy, gq[q][0] * w, gq[q][1] * w, gq[q][2] * w, Ts[qq] * d,
                                                 wx0 * wy0, wx1 * wy0, wx0 * wy1, wx1 * wy1);
                    }
                }
            }
        }
    }
}

// The box backward kernels by key (KeyTraits), and the deterministic ones (kKeyDet), which take the DetAcc too.
template <uint32_t K>
__global__ void __launch_bounds__(kBwdThreads, 1)
mpi_bwd_box_kernel(const RenderParams p, const __grid_constant__ TmaMaps maps, const int tiles_x, const int tiles_y) {
    static_assert((K & ~(kKeyAC | kKeyFac)) == (kKeyBwd | kKeyStaged), "a box backward key");
    bwd_box_body<KeyTraits<K>::kAlignCorners, KeyTraits<K>::kFactored, false>(p, maps, tiles_x, tiles_y, DetAcc{});
}

template <uint32_t K>
__global__ void __launch_bounds__(kBwdThreads, 1)
mpi_bwd_box_det_kernel(const RenderParams p, const __grid_constant__ TmaMaps maps, const int tiles_x, const int tiles_y, const DetAcc da) {
    static_assert((K & ~(kKeyAC | kKeyFac)) == (kKeyBwd | kKeyStaged | kKeyDet), "a deterministic box backward key");
    bwd_box_body<KeyTraits<K>::kAlignCorners, KeyTraits<K>::kFactored, true>(p, maps, tiles_x, tiles_y, da);
}

}  // namespace gmpi
