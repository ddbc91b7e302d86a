// Forward, TMA-staged persistent variant (the fast path).
//
// One CTA per SM walks (tile, plane) pairs: a 64x30-pixel output tile, planes front to back.  A producer warp computes,
// from the tile's four corner rays, the texel footprint of the tile on the next plane and issues cp.async.bulk.tensor
// copies of exactly that footprint (all four channels, rows in units of 4 issued as a few tall copies, origin aligned to 16 bytes,
// width rounded up to one of five compile-time classes) into a 2- or 3-stage shared-memory ring; 15 consumer warps (4 pixels = 2 pixel pairs per
// thread) take their 16 bilinear taps per pixel and plane from shared memory (a warp reads 32 consecutive x of one row:
// conflict-free while the texel/pixel scale is <= 1) and composite in registers.  TMA's out-of-bounds zero fill implements
// padding_mode="zeros".  Every consumer warp verifies (one vote) that all its taps lie inside the staged box; otherwise it
// takes the generic body, which checks each pixel and samples global memory where the box does not cover it, so results
// never depend on the footprint estimate (arbitrary ray tensors stay correct, only slower).  Tiles are walked full-height
// first, partial bottom tiles last (TileWalk).  DESIGN.md section 4.1 has the measurements and what bounds the kernel.
#pragma once
#include "mpi_common.cuh"
#include "tma_utils.cuh"
#include "mpi_kernel_keys.cuh"

namespace gmpi {

constexpr int kConsWarps = 15;   // 15 consumer warps + producer = 16 warps = 4 per scheduler, 128 registers per thread
constexpr int kPairs = 2;        // packed pixel pairs per thread (each pair = x and x+32 of one tile row)
constexpr int kPix = 2 * kPairs;
constexpr int kTileW = 64, kTileH = kPairs * kConsWarps;
constexpr int kConsThreads = kConsWarps * 32, kStagedThreads = kConsThreads + 32;
// Ring depth of the expanded forward, chosen at launch (fwd_ring_stages): kStages when the boxes come from L2, kStreamStages
// when they stream from HBM.  DESIGN.md section 4.1 has the measurements.
constexpr int kStages = 3, kStreamStages = 2;
constexpr int kRowsPerOp = 4;
constexpr int kMaxBW = 88;
constexpr int kMaxBH = (((kTileH * 5) / 4 + 6 + kRowsPerOp - 1) / kRowsPerOp) * kRowsPerOp;   // footprint rows at scale 1.25 + taps/slack, whole chunks
// Box widths are compile-time classes (multiples of 8: row pitch 4*bw = 0 mod 32 banks) so that the consumers'
// sixteen taps are LDS [reg + immediate]; the producer picks the narrowest class that covers the footprint.
constexpr int kMinBW = 56, kBWStep = 8;
constexpr int kNumMaps = (kMaxBW - kMinBW) / kBWStep + 1;
constexpr int kMaxPlanesStaged = 512;   // plane-constant table: 32 B per plane in shared memory
// Factored forward: box widths 64 and 96 only.  Its boxes are [row][3][bw] (colour) and [row][bw] (alpha): row pitches of 3 bw and
// bw words, and only a pitch that is a multiple of the 32 banks keeps a warp whose 32 taps straddle two texture rows (any rotated
// view) at one wavefront per LDS -- the expanded box [row][4][bw] has that for every bw % 8 == 0.  The 96-wide box holds footprints
// 65..kMaxBW texels wide: wider ones take the generic body, as in the expanded ring (see staged_producer).
constexpr int kWideBW = 96;

// Box width of class k (tensor-map slot k).  In the factored forward's ring (wide) slot 4 holds kWideBW and slot 1 the 64-wide boxes.
__host__ __device__ constexpr int class_width(int k, bool wide = false) { return wide && k == kNumMaps - 1 ? kWideBW : kMinBW + k * kBWStep; }

// MPI element types E (KeyTraits::Elem): fp32, fp16 (GMPI_MPI_F16) and uint8 (GMPI_MPI_U8, expanded only), each described once by
// ElemTraits<E>: ElemBase derives what follows from the element size, each specialisation states the rest.  TMA moves whole 16 bytes,
// so the tensor maps need Wt % kAlign == 0 and a staged box starts at a multiple of kAlign texels: the producer computes footprint,
// class, mode and box origin as in fp32 (a multiple of 4 texels), then stages the box at staged_origin(origin), staged_width(class
// width, factored) wide; StageMeta::sel bits 10-13 carry the offset between the two origins.  Class, mode and the in-box vote stay
// those of the fp32 box, so an MPI takes the fast and the generic body exactly where its fp32 conversion does.
template <class E, class B, CUtensorMapDataType kType>
struct ElemBase {
    using Elem = E;
    using Bits = B;                                         // an element's bit pattern
    static constexpr MapElem kMap = {kType, sizeof(E)};     // tensor-map data type and element bytes
    static constexpr int kAlign = 16 / sizeof(E);           // texels per 16 bytes
    // mask of the fp32 box's offset in the staged box: a compile-time 0 in fp32, whose boxes already start 16-byte aligned
    static constexpr int kOriginMask = kAlign == 4 ? 0 : kAlign - 1;
    static __host__ __device__ constexpr int staged_origin(int bx0) { return bx0 & ~kOriginMask; }
};
template <class E> struct ElemTraits;
// fp32.  Bit tests, shared by the range check and the occupancy build: non-finite = exponent all ones (inf, NaN); out of unit =
// outside [0, 1] and not -0.0 (negatives and NaN have larger patterns than 1.0).
template <> struct ElemTraits<float> : ElemBase<float, uint32_t, CU_TENSOR_MAP_DATA_TYPE_FLOAT32> {
    static __host__ __device__ constexpr int staged_width(int bw, bool) { return bw; }
    static __device__ __forceinline__ bool nonfinite(uint32_t b) { return (b & 0x7f800000u) == 0x7f800000u; }
    static __device__ __forceinline__ bool out_of_unit(uint32_t b) { return b > 0x3f800000u && b != 0x80000000u; }
};
// fp16: boxes start 0 or 4 texels west of the fp32 origin, so they are wider than their class: bw + 8 in the expanded ring; 96 and
// 128 for the factored ring's 64 and 96 (a colour copy of kColourCopyRows rows lands at a multiple of 132 bw bytes, which must be
// 128-byte aligned: bw % 32 == 0).  The bit tests give each half the verdict of its fp32 upcast.
template <> struct ElemTraits<__half> : ElemBase<__half, uint16_t, CU_TENSOR_MAP_DATA_TYPE_FLOAT16> {
    static __host__ __device__ constexpr int staged_width(int bw, bool factored) { return bw + (factored ? 32 : 8); }
    static __device__ __forceinline__ bool nonfinite(uint32_t b) { return (b & 0x7c00u) == 0x7c00u; }
    static __device__ __forceinline__ bool out_of_unit(uint32_t b) { return b > 0x3c00u && b != 0x8000u; }
};
// uint8 (expanded ring only): boxes start 0..12 texels west of the fp32 origin and are the 16-byte multiples that cover the class box
// after that shift: 80, 80, 96, 96, 112 for the classes 56 .. 88.  No bit tests: every code is finite and inside [0, 1].
template <> struct ElemTraits<uint8_t> : ElemBase<uint8_t, uint8_t, CU_TENSOR_MAP_DATA_TYPE_UINT8> {
    static __host__ __device__ constexpr int staged_width(int bw, bool) { return (bw + 12 + 15) & ~15; }
};

struct TmaMaps {
    CUtensorMap m[kNumMaps];      // expanded rgba [M*N][4][Ht][Wt] as (x, channel, y, plane), box {bw, 4, 4 rows, 1}
    CUtensorMap m8[kNumMaps], m16[kNumMaps], m32[kNumMaps];   // the same with 8-, 16- and 32-row boxes (see staged_producer: a
                                                              // footprint of r 4-row chunks goes out as the binary digits of r)
    // factored MPI: shared colour [M][3][Ht][Wt] as (x, channel, y, mpi), box {bw, 3, the ring's kColourCopyRows, 1}; the last
    // plane's own colour (torgba_sep_background) likewise; per-plane alpha [M*N][Ht][Wt] as (x, y, plane), box {bw, box height, 1}
    CUtensorMap rgb[kNumMaps], bg[kNumMaps], a[kNumMaps];
    CUtensorMap t;      // backward only: saved transmittance [V*N][H][W], box {64, 24, 1} (the backward's tile)
};

// per-stage header written by the producer before it arms the full barrier
struct __align__(16) StageMeta {
    int cx, cy;            // box origin (texel coordinates of smem element [0][.][0]) + kFloorMagicBits: bits(x + 1.5*2^23, rounded
                           // down) - cx is floor(x) relative to the box
    int rows2;             // staged rows - 2: a footprint with north-west tap (rx, ry) fits iff 0<=rx<=bw-2, 0<=ry<=rows-2
    int sel;               // bits 0-7 staged width (row pitch = 4*bw floats), bits 8-9 mode (0 staged, 1 nothing under the
                           // tile, 2 sample from global), bits 16-20 width class for the packed fast body, ONE-HOT (a chain of
                           // single-bit tests, most frequent first, is shorter than a jump table), or 0 (not usable: mode != 0,
                           // or plane constants outside the exact-division range, or -- backward only -- a footprint too
                           // magnified for the gradient box)
};

// ---- pixel-pair arithmetic: two pixels per operation, IEEE rn per element ----
// sm_90 has no packed fp32 instructions, so every pair operation is two scalar ones.  The explicitly rounded intrinsics
// (__fmul_rn, __fadd_rn, __fmaf_rn) are never contracted by the compiler, which keeps the reference's separately rounded
// mul-then-add (a contracted FFMA moves texel coordinates by a few ulp).
typedef float2 f2;
__device__ __forceinline__ f2 splat(float a) { return make_float2(a, a); }
__device__ __forceinline__ f2 mul2(f2 a, f2 b) { return make_float2(__fmul_rn(a.x, b.x), __fmul_rn(a.y, b.y)); }
__device__ __forceinline__ f2 add2(f2 a, f2 b) { return make_float2(__fadd_rn(a.x, b.x), __fadd_rn(a.y, b.y)); }
__device__ __forceinline__ f2 fma2(f2 a, f2 b, f2 c) { return make_float2(__fmaf_rn(a.x, b.x, c.x), __fmaf_rn(a.y, b.y, c.y)); }
// floor() without the XU pipe: t = x + 1.5*2^23 rounded toward -inf has floor(x) in its mantissa (exact for |x| < 2^22):
// floor as float = t - 1.5*2^23, floor as int = bits(t) - 0x4b400000.  Anything out of range (huge, inf, NaN) yields an
// integer far outside any staged box, so the unsigned box test rejects it.
__device__ __forceinline__ f2 add2_rm(f2 a, f2 b) { return make_float2(__fadd_rd(a.x, b.x), __fadd_rd(a.y, b.y)); }
constexpr float kFloorMagic = 12582912.0f;        // 1.5 * 2^23
constexpr int kFloorMagicBits = 0x4b400000;
constexpr int kSelSlow = 0;     // class field is one-hot (bit 16 + class); 0 = packed fast body not usable

// a / b correctly rounded with y = RN(1/b), nb = -b (div_by_rcp, two pixels at once)
__device__ __forceinline__ f2 div2_by_rcp(f2 a, f2 nb, f2 y) {
    const f2 q0 = mul2(a, y);
    const f2 r = fma2(q0, nb, a);
    return fma2(r, y, q0);
}

// A thread's four pixels as two pairs: pair P = (x = lane, x = lane + 32) on tile row 2*warp + P.
struct RayPairs {
    f2 rx2[kPairs], ry2[kPairs];   // 2*ray_x, 2*ray_y
    f2 nrz[kPairs], yrz[kPairs];   // -ray_z, RN(1/ray_z)
};
__device__ __forceinline__ void pack_ray_pairs(const RayConst (&rc)[kPix], RayPairs& rp) {
#pragma unroll
    for (int P = 0; P < kPairs; ++P) {
        rp.rx2[P] = make_float2(rc[2 * P].rx2, rc[2 * P + 1].rx2);
        rp.ry2[P] = make_float2(rc[2 * P].ry2, rc[2 * P + 1].ry2);
        rp.nrz[P] = make_float2(-rc[2 * P].rz, -rc[2 * P + 1].rz);
        rp.yrz[P] = make_float2(rc[2 * P].yrz, rc[2 * P + 1].yrz);
    }
}
struct CoordPairs {
    f2 ix[kPairs], iy[kPairs], sc[kPairs];
};

// Texel coordinates on one plane, exact-division fast form; op order of plane_coord (mpi.py:74-90 + unnormalize).
template <bool kAlignCorners>
__device__ __forceinline__ void coords_pairs(const PlaneConst& pc, const RayPairs& rp, f2 ex2, f2 ey2, f2 hsx, f2 hsy, float fWt,
                                             float fHt, CoordPairs& c) {
    const f2 zd = splat(pc.z_diff), ypw = splat(pc.ypw), yph = splat(pc.yph), npw = splat(-pc.pw), nph = splat(-pc.ph);
    const f2 one = splat(1.0f);
#pragma unroll
    for (int P = 0; P < kPairs; ++P) {
        const f2 sq = div2_by_rcp(zd, rp.nrz[P], rp.yrz[P]);                 // scale = z_diff / ray_z
        // 2*(e_x + ray_x*scale): mul, THEN add (two roundings, mpi.py:79); __fmul_rn/__fadd_rn are never contracted
        const f2 X2 = make_float2(__fadd_rn(ex2.x, __fmul_rn(rp.rx2[P].x, sq.x)), __fadd_rn(ex2.y, __fmul_rn(rp.rx2[P].y, sq.y)));
        const f2 Y2 = make_float2(__fadd_rn(ey2.x, __fmul_rn(rp.ry2[P].x, sq.x)), __fadd_rn(ey2.y, __fmul_rn(rp.ry2[P].y, sq.y)));
        f2 u = div2_by_rcp(X2, npw, ypw);                                    // (2x) / width
        f2 v = div2_by_rcp(Y2, nph, yph);
        if (kAlignCorners) {
            c.ix[P] = mul2(add2(u, one), hsx);                               // (u+1) * ((Wt-1)/2)
            c.iy[P] = mul2(add2(v, one), hsy);
        } else {
            if (u.x >= -1.0f && u.x <= 1.0f) u.x = __fmul_rn(u.x, 0.95f);
            if (u.y >= -1.0f && u.y <= 1.0f) u.y = __fmul_rn(u.y, 0.95f);
            if (v.x >= -1.0f && v.x <= 1.0f) v.x = __fmul_rn(v.x, 0.95f);
            if (v.y >= -1.0f && v.y <= 1.0f) v.y = __fmul_rn(v.y, 0.95f);
            const f2 half = splat(0.5f), m1 = splat(-1.0f);
            c.ix[P] = mul2(add2(mul2(add2(u, one), splat(fWt)), m1), half);  // ((u+1)*W - 1) / 2
            c.iy[P] = mul2(add2(mul2(add2(v, one), splat(fHt)), m1), half);
        }
        c.sc[P] = sq;
    }
}

// The bilinear footprints of a thread's two pixel pairs in a staged box of compile-time width BW, shared by the forward's and
// the backward's fast bodies.  AOFF == 0: expanded stage [row][4 channels][BW].  AOFF > 0 (factored MPI): colour box [row][3][BW]
// at the stage base and the alpha box [row][BW] AOFF floats further on.  The backward's gradient box has the stage's layout, so
// the same indices address it.  E: the element type of the box (fp16 boxes under GMPI_MPI_F16: each tap is converted to fp32).
template <int BW, int AOFF, class E = float>
struct BoxTaps {
    static constexpr int SW = ElemTraits<E>::staged_width(BW, AOFF != 0);   // staged box width (BW: the box the vote tests)
    static constexpr int RP = AOFF ? 3 * SW : 4 * SW;       // colour row pitch
    static constexpr int AP = AOFF ? SW : 4 * SW;           // alpha row pitch
    static constexpr int A0 = AOFF ? AOFF : 3 * SW;         // alpha offset from the colour index (factored: separate box)
    f2 fx0[kPairs], fy0[kPairs];                            // floor of the coordinates, as floats
    int ia[kPairs], ib[kPairs];                             // colour index of the north-west taps of pixels .x and .y of pair P
    int ja[kPairs], jb[kPairs];                             // factored: alpha index (separate box)

    // Floors and indices of every footprint.  Returns the warp's vote that all of them lie inside the box (warp-uniform, so the
    // caller's fallback needs no reconvergence scaffolding).
    __device__ __forceinline__ bool locate(int cx, int cy, int rows2, const CoordPairs& c) {
        const f2 magic = splat(kFloorMagic), nmagic = splat(-kFloorMagic);
        bool inbox = true;
#pragma unroll
        for (int P = 0; P < kPairs; ++P) {
            const f2 tx = add2_rm(c.ix[P], magic), ty = add2_rm(c.iy[P], magic);         // floor without the XU pipe
            fx0[P] = add2(tx, nmagic);                                    // floor as float (exact)
            fy0[P] = add2(ty, nmagic);
            const int rxa = __float_as_int(tx.x) - cx, rxb = __float_as_int(tx.y) - cx;   // floor - box origin, as integers
            const int rya = __float_as_int(ty.x) - cy, ryb = __float_as_int(ty.y) - cy;
            inbox = inbox && (unsigned)rxa <= (unsigned)(BW - 2) && (unsigned)rxb <= (unsigned)(BW - 2) &&
                    (unsigned)rya <= (unsigned)rows2 && (unsigned)ryb <= (unsigned)rows2;
            ia[P] = rya * RP + rxa;                                       // [row][channel][x], compile-time pitch
            ib[P] = ryb * RP + rxb;
            if (AOFF) { ja[P] = rya * AP + rxa + A0; jb[P] = ryb * AP + rxb + A0; }
        }
        return __all_sync(0xffffffffu, inbox);
    }
    // one channel of pair P: the four taps of a box with row pitch PITCH at ta / tb, weighted
    template <int PITCH>
    static __device__ __forceinline__ f2 tap2(const E* ta, const E* tb, const f2 (&w)[4]) {
        return fma2(make_float2(to_f32(ta[PITCH + 1]), to_f32(tb[PITCH + 1])), w[3],
                    fma2(make_float2(to_f32(ta[PITCH]), to_f32(tb[PITCH])), w[2],
                         fma2(make_float2(to_f32(ta[1]), to_f32(tb[1])), w[1], mul2(make_float2(to_f32(ta[0]), to_f32(tb[0])), w[0]))));
    }
    // bilinear weights w = (w00, w01, w10, w11) and the four channels of pair P from the staged box sb
    __device__ __forceinline__ void sample(const E* __restrict__ sb, const CoordPairs& c, int P, f2 (&w)[4], f2& r, f2& g, f2& b,
                                           f2& a) const {
        const f2 m1 = splat(-1.0f), one = splat(1.0f);
        const f2 wx1 = fma2(fx0[P], m1, c.ix[P]), wy1 = fma2(fy0[P], m1, c.iy[P]);   // fractional parts (exact)
        const f2 wy0 = fma2(wy1, m1, one);
        w[3] = mul2(wx1, wy1); w[2] = fma2(w[3], m1, wy1); w[1] = fma2(w[3], m1, wx1); w[0] = fma2(w[1], m1, wy0);
        const E* ta = sb + ia[P];
        const E* tb = sb + ib[P];
        r = tap2<RP>(ta, tb, w);
        g = tap2<RP>(ta + SW, tb + SW, w);
        b = tap2<RP>(ta + 2 * SW, tb + 2 * SW, w);
        a = AOFF ? tap2<AP>(sb + ja[P], sb + jb[P], w) : tap2<AP>(ta + A0, tb + A0, w);
    }
};

// Sample + composite the four pixels from a staged box of compile-time width BW.  Returns false (and changes nothing)
// if any of the four footprints is not inside the box.  AOFF as in BoxTaps.
// kES (early stop): a pixel whose |T| <= tau adds nothing; its weight is selected to 0, so its T stays where it stopped.
template <int BW, int AOFF = 0, bool kES = false, class E = float>
__device__ __forceinline__ bool sample_pairs(const E* __restrict__ sb, int cx, int cy, int rows2, const CoordPairs& c,
                                             f2 (&T)[kPairs], f2 (&cr)[kPairs], f2 (&cg)[kPairs], f2 (&cb)[kPairs], f2 (&cws)[kPairs],
                                             float tau = 0.0f) {
    const f2 m1 = splat(-1.0f);
    BoxTaps<BW, AOFF, E> bt;
    if (!bt.locate(cx, cy, rows2, c)) return false;
#pragma unroll
    for (int P = 0; P < kPairs; ++P) {
        f2 wb[4], r, g, b, a;
        bt.sample(sb, c, P, wb, r, g, b, a);
        f2 w = mul2(a, T[P]);                           // mpi.py:423
        if (kES) {
            if (fabsf(T[P].x) <= tau) w.x = 0.0f;
            if (fabsf(T[P].y) <= tau) w.y = 0.0f;
        }
        cr[P] = fma2(w, r, cr[P]);                      // mpi.py:430
        cg[P] = fma2(w, g, cg[P]);
        cb[P] = fma2(w, b, cb[P]);
        cws[P] = fma2(w, c.sc[P], cws[P]);              // depth_i = scale * (ray . z_dir), mpi.py:150
        T[P] = fma2(w, m1, T[P]);   // T(1-a); the reference's +1e-10 changes any later weight by < 1e-10 absolute
    }
    return true;
}

// Rare path (a ray whose footprint is not in the staged box): sample the plane from global memory.  Out of line so
// that it does not cost registers in the hot loop.
// Expanded MPI: ONE base pointer crosses the call.  (Passing the four channel pointers of PlaneChans instead -- 8 registers that
// are live only inside the rare branch -- still shifted the register allocation of the hot loop: -3.8 % frames/s, bisected on
// the GPU in round 2.  The factored instantiation, which needs them, is a separate template instance.)
// Three translation units of the one library define the four non-template overloads.  Their host stubs are static, so that the
// library links; their device code keeps external linkage, because static device functions change where ptxas places the
// deterministic box backward's subroutines, and so that kernel's machine code.
#ifdef __CUDA_ARCH__
#define GMPI_HOST_STATIC
#else
#define GMPI_HOST_STATIC static
#endif
GMPI_HOST_STATIC __device__ __noinline__ float4 sample_plane_direct(const float* __restrict__ plane, int Ht, int Wt, float ix, float iy) {
    const size_t tex = (size_t)Ht * Wt;
    const Taps tp = make_taps(ix, iy, Ht, Wt);
    return make_float4(tap4(plane, tp), tap4(plane + tex, tp), tap4(plane + 2 * tex, tp), tap4(plane + 3 * tex, tp));
}
GMPI_HOST_STATIC __device__ __noinline__ float4 sample_chans_direct(const PlaneChans pl, int Ht, int Wt, float ix, float iy) {
    const Taps tp = make_taps(ix, iy, Ht, Wt);
    return make_float4(tap4(pl.c[0], tp), tap4(pl.c[1], tp), tap4(pl.c[2], tp), tap4(pl.c[3], tp));
}
// the same from an fp16 MPI (overloads, so that the fp32 functions keep their symbols)
GMPI_HOST_STATIC __device__ __noinline__ float4 sample_plane_direct(const __half* __restrict__ plane, int Ht, int Wt, float ix, float iy) {
    const size_t tex = (size_t)Ht * Wt;
    const Taps tp = make_taps(ix, iy, Ht, Wt);
    return make_float4(tap4(plane, tp), tap4(plane + tex, tp), tap4(plane + 2 * tex, tp), tap4(plane + 3 * tex, tp));
}
GMPI_HOST_STATIC __device__ __noinline__ float4 sample_chans_direct(const PlaneChansT<__half> pl, int Ht, int Wt, float ix, float iy) {
    const Taps tp = make_taps(ix, iy, Ht, Wt);
    return make_float4(tap4(pl.c[0], tp), tap4(pl.c[1], tp), tap4(pl.c[2], tp), tap4(pl.c[3], tp));
}
// any other element type (uint8_t, GMPI_MPI_U8): templates, instantiated only by the kernels that use them (mpi_u8.cu); the overloads
// above stay the exact matches for fp32 and fp16
template <class E>
__device__ __noinline__ float4 sample_plane_direct(const E* __restrict__ plane, int Ht, int Wt, float ix, float iy) {
    const size_t tex = (size_t)Ht * Wt;
    const Taps tp = make_taps(ix, iy, Ht, Wt);
    return make_float4(tap4(plane, tp), tap4(plane + tex, tp), tap4(plane + 2 * tex, tp), tap4(plane + 3 * tex, tp));
}
template <class E>
__device__ __noinline__ float4 sample_chans_direct(const PlaneChansT<E> pl, int Ht, int Wt, float ix, float iy) {
    const Taps tp = make_taps(ix, iy, Ht, Wt);
    return make_float4(tap4(pl.c[0], tp), tap4(pl.c[1], tp), tap4(pl.c[2], tp), tap4(pl.c[3], tp));
}
// generic-path sample of plane i of MPI m: the instantiation decides which form crosses the call
template <bool kFactored, class E>
__device__ __forceinline__ float4 sample_plane_any(const RenderParams& p, const E* plane, int m, int i, size_t tex, float ix, float iy) {
    if (kFactored) return sample_chans_direct(plane_chans<E>(p, m, i, tex), p.Ht, p.Wt, ix, iy);
    return sample_plane_direct(plane, p.Ht, p.Wt, ix, iy);
}

// named barrier 1 over the kThreads consumer threads of a kernel
template <int kThreads>
__device__ __forceinline__ void consumer_bar_sync() { asm volatile("bar.sync 1, %0;" ::"n"(kThreads) : "memory"); }

// Tile order of the persistent grid (producer and consumers walk the same sequence): every full-height tile of every view
// first, round-robin over the CTAs; then the partial bottom-row tiles (H % kTileH valid rows), dealt only to the CTAs that
// got one full tile fewer.  Warps whose rows lie outside the image only keep the ring protocol going, so a partial tile
// costs a fraction of a full one and fills the last, incomplete round of the grid instead of stretching it
// (96 planes, 1024^2 x 4 views on 132 SMs: 2176 full tiles = 16 rounds + 64, and the 64 partial tiles go to the 68 CTAs
// that got 16).
struct TileXY { int v, px0, py0; };
struct TileWalk {
    int tiles_x, full_rows, full_per_view, n_full, n_part;
    int cta, grid;               // blockIdx.x, gridDim.x (members so that the host-side test hook runs the same code)
    int n1, p_start, p_step;     // this CTA: number of full tiles; first partial tile and stride (p_step == 0: none)
    int tile_h;                  // tile height in pixels (forward: kTileH = 30, backward: 24)
    int group;                   // views per MPI when consecutive views share one (1: order tiles view by view).  With
                                 // group > 1 the views of a group are the FASTEST index: the CTAs running at the same time
                                 // work on the same tile position of different views of one MPI, i.e. on (nearly) the same
                                 // texels, which then come from L2 instead of HBM (video render: 120 views of one MPI)
    // (lives in shared memory, filled by one thread: it is read once per tile and must not cost registers in the plane loop)
    __host__ __device__ __forceinline__ void init(int tiles_x_, int H, int V, int cta_, int grid_, int tile_h_ = kTileH, int group_ = 1) {
        tiles_x = tiles_x_;
        cta = cta_; grid = grid_;
        tile_h = tile_h_;
        group = (group_ > 1 && V % group_ == 0) ? group_ : 1;
        full_rows = H / tile_h;
        full_per_view = tiles_x * full_rows;
        n_full = full_per_view * V;
        n_part = (H % tile_h) ? tiles_x * V : 0;
        const int b = cta, G = grid, r = n_full % G;
        n1 = b < n_full ? (n_full - b + G - 1) / G : 0;
        if (r == 0) { p_start = b; p_step = G; }
        else if (b >= r) { p_start = b - r; p_step = G - r; }
        else { p_start = 0; p_step = 0; }
    }
    // index t of a sequence of `per_view` positions x V views -> (view, position): view-major, or group-minor
    __host__ __device__ __forceinline__ void split(int t, int per_view, int& v, int& pos) const {
        if (group == 1) { v = t / per_view; pos = t - v * per_view; return; }
        const int per_group = per_view * group, g = t / per_group, rem = t - g * per_group;
        pos = rem / group;
        v = g * group + (rem - pos * group);
    }
    // j-th tile of this CTA; false when done
    __host__ __device__ __forceinline__ bool at(int j, TileXY& r) const {
        int pos;
        if (j < n1) {
            split(cta + j * grid, full_per_view, r.v, pos);
            r.px0 = (pos % tiles_x) * kTileW; r.py0 = (pos / tiles_x) * tile_h;
            return true;
        }
        if (p_step == 0) return false;
        const int u = p_start + (j - n1) * p_step;
        if (u >= n_part) return false;
        split(u, tiles_x, r.v, pos);
        r.px0 = pos * kTileW; r.py0 = full_rows * tile_h;
        return true;
    }
};

// A consumer warp without a single row inside the image: hand every stage of this tile straight back to the producer.
__device__ __forceinline__ void consumer_idle_tile(uint64_t* s_full, uint64_t* s_empty, int N, int n_stages, int lane, int& c_stage,
                                                   uint32_t& c_phase) {
    for (int i = 0; i < N; ++i) {
        const int s = c_stage;
        const uint32_t ph = c_phase;
        if (++c_stage == n_stages) { c_stage = 0; c_phase ^= 1u; }
        mbar_wait(&s_full[s], ph);
        __syncwarp();
        mbar_arrive_if(&s_empty[s], lane == 0);
    }
}

// Ring geometry of a kernel: tile height, ring depth, the largest staged box and what a stage holds.
// The staged forward's ring on an MPI of element type E: expanded, or (kFactored) the factored forward's 64- or 96-wide boxes (see
// kWideBW).  A stage holds the staged box (ElemTraits) of the widest class.
template <bool kFactored, class E>
struct FwdRing {
    static constexpr int kTileRows = kTileH, kRingStages = kStages, kBoxMaxH = kMaxBH;
    // elements of one staged plane box, and per ring stage
    static constexpr int kPlaneFloats = ElemTraits<E>::staged_width(kFactored ? kWideBW : kMaxBW, kFactored) * kMaxBH * 4;
    static constexpr int kStride = kPlaneFloats;
    static constexpr size_t kStageBytes = (size_t)kPlaneFloats * sizeof(E);
    static constexpr bool kReverse = false;                // planes front to back; no transmittance box
    // producer sleeps between polls of a full ring (see mbar_wait_sleep).  Measured: sleeping costs the forward 1 % (a shallow
    // ring wants its producer prompt)
    static constexpr bool kSleepPolls = false;
    static constexpr bool kWideFact = kFactored;
    static constexpr bool kBinaryCopies = true;            // expanded MPI: copies of 32/16/8/4 rows (see staged_producer)
    // factored MPI: colour box = 2 copies of 22 rows.  A copy lands at row offset r * 3 * bw * sizeof(E) bytes, which must be a
    // multiple of 128 (TMA destination alignment): any r for the staged widths 64 / 96 in fp32, 96 / 128 in fp16.
    static constexpr int kColourCopyRows = kMaxBH / 2;
    static_assert(kStages * kStageBytes + (size_t)kMaxPlanesStaged * 32 + 1024 <= 227 * 1024, "the ring must fit one SM");
};
static_assert(kMaxBH % 2 == 0 && kMaxBH / kRowsPerOp < 16, "half-height colour copies; binary digits of the chunk count");
static_assert(FwdRing<false, float>::kPlaneFloats == 15488 && FwdRing<true, float>::kPlaneFloats == 16896 &&
              FwdRing<false, __half>::kPlaneFloats == 16896 && FwdRing<true, __half>::kPlaneFloats == 22528 &&
              FwdRing<false, uint8_t>::kPlaneFloats == 19712, "the staged forward's ring stages");
// uint8: a multiple of 128 bytes, so that every stage and every 4-row copy (16 * staged width bytes per chunk) lands 128-byte aligned
static_assert(FwdRing<false, uint8_t>::kStageBytes % 128 == 0, "uint8 ring stages stay 128-byte aligned");

// The expanded forward's copies of one stage: the footprint's n_chunks 4-row chunks as the binary digits of n_chunks.  Lane 0..3
// owns the digit 8, 4, 2, 1: returns the copy's height in chunks (0: this lane issues nothing) and, in `before`, the chunks
// covered by the taller copies, i.e. where this copy starts.  (Host-evaluable: gmpi_debug_copy_plan, tests/test_tile_walk.py.)
__host__ __device__ __forceinline__ int binary_copy_of_lane(int n_chunks, int lane, int& before) {
    const int bit = 3 - lane;
    before = (n_chunks >> (bit + 1)) << (bit + 1);
    return ((n_chunks >> bit) & 1) << bit;
}

// Early stop (kES, forward only).  s_stop[j % kStopSlots] holds one bit per consumer warp that has stopped in the CTA's j-th tile.
// The producer sets it to the warps without a row in the image when it arms the tile's first stage; a consumer warp ORs its bit
// in once all its pixels have stopped, before it releases the stage it stopped on.  Before each later stage of the tile the
// producer reads the word, and when every warp has stopped it arms the stage without copies (mbar_arrive, no transaction
// bytes): the ring's sequence of stages and phases is unchanged, only the TMA traffic goes.  A read that misses a bit costs one
// box that nobody samples; a set bit is always true, so results never depend on timing.  Slots: the producer runs at most
// n_stages - 1 stages ahead of the slowest consumer, i.e. at most 1 + (n_stages - 1) / N tiles ahead (3 for N = 1 and a
// 3-stage ring), so a slot is not reset while a consumer of its previous tile could still write it.
constexpr int kStopSlots = 4;
constexpr uint32_t kAllConsumers = (1u << kConsWarps) - 1u;
static_assert(kStages <= kStopSlots, "stop-word slots must cover the producer's lead");
__device__ unsigned long long g_early_stop_skipped;   // test hook: stages armed without copies (gmpi_debug_fwd_early_stop_stats)

// Empty-space skipping (kSkip, forward only, mpi_fwd_skip_kernel).  The occupancy map has one bit per kOccB x kOccB texel
// block of every (MPI, plane), set when a texel of the block is not empty: alpha is not +0 (bit pattern 0), or a colour value is
// not finite.  A plane's map is `rows` block rows of `words` 32-bit words (bit b of word w: block column 32 w + b).  Compositing a
// box whose texels are all empty adds fma(+0, finite, x) == x to every sum and leaves T alone, so the producer arms such a stage
// without copies and marks it kSelEmpty; consumers composite nothing where their taps fall in the box (DESIGN.md section 4.1).
constexpr int kOccB = 8;
constexpr int kSelEmpty = 1 << 24;      // StageMeta::sel: the stage's box is empty and was not loaded
struct OccMap {
    const uint32_t* bits;           // [M*N][rows][words]
    int words, rows;
    unsigned long long* skipped;    // stats: stages armed empty (gmpi_debug_fwd_skip_stats)
};
__host__ __device__ __forceinline__ int occ_words(int Wt) { return ((Wt + kOccB - 1) / kOccB + 31) / 32; }
__host__ __device__ __forceinline__ int occ_rows(int Ht) { return (Ht + kOccB - 1) / kOccB; }

// The map builds (mpi_skip.cu, mpi_u8.cu): one CTA row of kOccThreads threads = 256 texel columns = one map word per plane.
constexpr int kOccThreads = 32 * kOccB;

// The 256 threads' verdicts (texel column threadIdx.x of this word is occupied) -> the map word: each warp holds 4 blocks of 8 columns.
__device__ __forceinline__ void store_occ_word(bool occupied, uint32_t* dst, uint32_t* s_w) {
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const uint32_t b = __ballot_sync(0xffffffffu, occupied);
    const uint32_t nib = ((b & 0xffu) ? 1u : 0u) | ((b & 0xff00u) ? 2u : 0u) | ((b & 0xff0000u) ? 4u : 0u) | ((b & 0xff000000u) ? 8u : 0u);
    if (lane == 0) s_w[warp] = nib << (4 * warp);
    __syncthreads();
    if (threadIdx.x == 0) {
        uint32_t w = 0;
#pragma unroll
        for (int k = 0; k < kOccThreads / 32; ++k) w |= s_w[k];
        *dst = w;
    }
    __syncthreads();
}

// Lane `lane`'s part of the box-versus-map test: the OR of the map bits of one plane under the texels [bx0, bx0 + bw) x
// [by0, by0 + rows) that lie inside the texture (TMA zero-fills the rest).  The (block row, word) pairs under the box are dealt to
// lanes lane, lane + 32, ... (a staged box covers at most 7 block rows of 2 words).  The box is empty iff no lane returns a bit.
// (Host-evaluable: gmpi_debug_box_occupied, tests/test_skip_empty.py.)
__host__ __device__ __forceinline__ uint32_t occ_box_bits(const uint32_t* plane, int Ht, int Wt, int words, int bx0, int by0, int bw,
                                                          int rows, int lane) {
    const int x0 = max(bx0, 0), x1 = min(bx0 + bw - 1, Wt - 1), y0 = max(by0, 0), y1 = min(by0 + rows - 1, Ht - 1);
    if (x0 > x1 || y0 > y1) return 0u;
    const int c0 = x0 / kOccB, c1 = x1 / kOccB, r0 = y0 / kOccB, r1 = y1 / kOccB;
    const int w0 = c0 >> 5, nw = (c1 >> 5) - w0 + 1, n = (r1 - r0 + 1) * nw;
    uint32_t acc = 0u;
    for (int l = lane; l < n; l += 32) {
        const int r = r0 + l / nw, w = w0 + l % nw;
        const int lo = max(c0 - 32 * w, 0), hi = min(c1 - 32 * w, 31);
#ifdef __CUDA_ARCH__
        const uint32_t word = __ldg(plane + (size_t)r * words + w);
#else
        const uint32_t word = plane[(size_t)r * words + w];
#endif
        acc |= word & (0xffffffffu >> (31 - hi)) & (0xffffffffu << lo);
    }
    return acc;
}

// The fast body's in-box vote (BoxTaps::locate) for a stage the producer marked empty: every footprint of the warp has its north-west
// tap at 0 <= rx <= bw2, 0 <= ry <= rows2 relative to the box.
__device__ __forceinline__ bool box_vote(int cx, int cy, int bw2, int rows2, const CoordPairs& c) {
    const f2 magic = splat(kFloorMagic);
    bool inbox = true;
#pragma unroll
    for (int P = 0; P < kPairs; ++P) {
        const f2 tx = add2_rm(c.ix[P], magic), ty = add2_rm(c.iy[P], magic);
        inbox = inbox && (unsigned)(__float_as_int(tx.x) - cx) <= (unsigned)bw2 && (unsigned)(__float_as_int(tx.y) - cx) <= (unsigned)bw2 &&
                (unsigned)(__float_as_int(ty.x) - cy) <= (unsigned)rows2 && (unsigned)(__float_as_int(ty.y) - cy) <= (unsigned)rows2;
    }
    return __all_sync(0xffffffffu, inbox);
}

// consumer warps of a tile at row py0 without a row inside an image of H rows (they only keep the ring going)
__device__ __forceinline__ uint32_t idle_consumer_warps(int py0, int H) {
    const int live = (H - py0 + kPairs - 1) / kPairs;
    return live >= kConsWarps ? 0u : kAllConsumers & ~((1u << live) - 1u);
}

// Producer warp, shared by the forward (front-to-back) and backward (back-to-front) kernels: for every (tile, plane) of
// this CTA, estimate the tile's texel footprint from its four corner rays, pick the narrowest box class, publish the stage
// header and issue the TMA copies.
// kFact: factored MPI (compile time: a run-time test of p.alpha in this loop cost the forward 1 %, the producer's per-stage latency
// being on the critical path of a shallow ring).
// E: the MPI's element type (the ring holds boxes of it).
// kSkip: empty-space skipping against the occupancy map `occ` (forward only, see OccMap).
template <bool kAlignCorners, class Ring, bool kFact, bool kES = false, class E = float, bool kSkip = false>
__device__ __forceinline__ void staged_producer(const RenderParams& p, const TmaMaps& maps, E* s_buf, StageMeta* s_meta,
                                            uint64_t* s_full, uint64_t* s_empty, const TileWalk* s_walk, int lane,
                                            int n_stages = Ring::kRingStages, uint32_t* s_stop = nullptr, OccMap occ = OccMap{}) {
    constexpr bool kReverse = Ring::kReverse;
    constexpr int kStride = Ring::kStride;      // floats per ring stage
    constexpr int kTileH = Ring::kTileRows, kMaxBH = Ring::kBoxMaxH, kStageFloats = Ring::kPlaneFloats;
    constexpr uint32_t kTBytes = kReverse ? (uint32_t)(kTileW * kTileH * 4) : 0u;
    const int Ht = p.Ht, Wt = p.Wt, N = p.N;
    const float fWt = (float)Wt, fHt = (float)Ht;
    const float hsx = 0.5f * (float)(Wt - 1), hsy = 0.5f * (float)(Ht - 1);
    const size_t img = (size_t)p.H * p.W;
    if (lane < kNumMaps) {
        if (kFact) { tma_prefetch_desc(&maps.rgb[lane]); tma_prefetch_desc(&maps.a[lane]); }
        else { tma_prefetch_desc(&maps.m[lane]); tma_prefetch_desc(&maps.m8[lane]); tma_prefetch_desc(&maps.m16[lane]); tma_prefetch_desc(&maps.m32[lane]); }
    }
    int p_stage = 0;
    uint32_t p_phase = 0;
    uint32_t n_skipped = 0;      // kES: stages armed without copies
    uint32_t n_empty = 0;        // kSkip: stages armed empty
    TileXY txy;
    for (int j = 0; s_walk->at(j, txy); ++j) {
        const int v = txy.v, px0 = txy.px0, py0 = txy.py0;
        const int m = __ldg(p.view2mpi + v);
        uint32_t* const stop_word = kES ? s_stop + (j & (kStopSlots - 1)) : nullptr;
        float ev[3], zd[3];
        load_eye_z(p, v, ev, zd);
        // the four corner pixels of the tile (replicated over the warp), clamped into the image
        const int cx = min(px0 + ((lane & 1) ? kTileW - 1 : 0), p.W - 1);
        const int cy = min(py0 + ((lane & 2) ? kTileH - 1 : 0), p.H - 1);
        float crx, cry, crz;
        load_ray(p, v, cx, cy, img, crx, cry, crz);
        const RayConst rc = make_ray_const(crx, cry, crz, ev, zd);
        for (int ii = 0; ii < N; ++ii) {
            const int i = kReverse ? N - 1 - ii : ii;
            const int s = p_stage;
            const uint32_t ph = p_phase;
            if (++p_stage == n_stages) { p_stage = 0; p_phase ^= 1u; }
            const PlaneConst pc = make_plane_const(p.dhw + ((size_t)m * N + i) * 3, ev[2]);
            const TexCoord tc = plane_coord<kAlignCorners>(pc, rc, hsx, hsy, fWt, fHt);
            // footprint of the tile = bounding box of the corner coordinates (the pixel -> texel map is projective,
            // hence monotone along image rows and columns), +-1 texel of slack for rounding
            const bool finite = fabsf(tc.ix) < 1e9f && fabsf(tc.iy) < 1e9f;
            const bool all_finite = __all_sync(0xffffffffu, finite);
            const int fx = finite ? (int)floorf(tc.ix) : 0, fy = finite ? (int)floorf(tc.iy) : 0;
            const int xmin = __reduce_min_sync(0xffffffffu, fx), xmax = __reduce_max_sync(0xffffffffu, fx);
            const int ymin = __reduce_min_sync(0xffffffffu, fy), ymax = __reduce_max_sync(0xffffffffu, fy);
            // TMA needs a 16-byte aligned start in the innermost dimension: the box origin is a multiple of 4 texels (fp16: the staged
            // box starts at bxs, a multiple of 8, uint8: of 16, see ElemTraits)
            const int bx0 = ((xmin - 1) >> 2) << 2, by0 = ymin - 1;
            const int need_w = xmax - bx0 + 3, need_h = ymax - ymin + 4;      // +1 east/south tap, +-1 slack
            int mode = 0;
            constexpr bool kWide = kFact && Ring::kWideFact;
            // Footprints wider than kMaxBW take the generic body in every ring, the factored forward's 96-wide boxes included: the fast
            // body forms its bilinear weights as w10 = wy1 - wx1 wy1 (FMAs), the generic body as (1 - wx1) wy1, which differ in the
            // last bit, so a footprint 89..96 texels wide staged here but not in the expanded ring would break the factored render's
            // bitwise equality with the expanded one.
            if (!all_finite || need_w > kMaxBW || ((need_h + kRowsPerOp - 1) / kRowsPerOp) * kRowsPerOp > kMaxBH) mode = 2;   // would not fit a ring stage
            else if (bx0 > Wt - 1 || bx0 + need_w - 1 < 0 || by0 > Ht - 1 || by0 + need_h - 1 < 0) mode = 1;
            // width class k (tensor-map slot, one-hot bit 16 + k of the header); wide rings: slot 1 = 64, slot 4 = kWideBW
            const int k = mode != 0 ? 0 : kWide ? (need_w <= 64 ? 1 : 4) : max(0, (need_w - kMinBW + kBWStep - 1) / kBWStep);
            const int bw = class_width(k, kWide);
            const int bxs = ElemTraits<E>::staged_origin(bx0), sw = ElemTraits<E>::staged_width(bw, kWide);   // staged box: origin, width
            const int n_ops = mode == 0 ? (need_h + kRowsPerOp - 1) / kRowsPerOp : 0;
            const int rows = n_ops * kRowsPerOp;
            // kSkip: only a stage that takes the fast body (mode 0, plane constants in the exact range) may be skipped.  The test covers
            // the whole box the consumers' in-box test accepts (class width bw, not need_w).  Its map loads are issued before the wait
            // for a free stage and voted on after it, so that their latency hides behind the wait.  (Probing one plane ahead, which
            // repeats the box computation, made the producer slower still: DESIGN.md section 4.1.)
            const bool testable = kSkip && mode == 0 && pc.fast != 0.0f;
            uint32_t occ_bits = 0u;
            if (testable) occ_bits = occ_box_bits(occ.bits + ((size_t)m * N + i) * occ.rows * occ.words, Ht, Wt, occ.words, bx0, by0, bw, rows, lane);
            if (Ring::kSleepPolls) mbar_wait_sleep(&s_empty[s], ph ^ 1);
            else mbar_wait(&s_empty[s], ph ^ 1);
            bool empty = false;
            if constexpr (kSkip) {
                empty = testable && !__any_sync(0xffffffffu, occ_bits != 0u);
                n_empty += empty ? 1u : 0u;
            }
            bool skip = false;
            if constexpr (kES) {
                if (ii == 0) {
                    if (lane == 0) *stop_word = idle_consumer_warps(py0, p.H);   // published by the full barrier's arrive below
                } else {
                    skip = __shfl_sync(0xffffffffu, *(volatile uint32_t*)stop_word, 0) == kAllConsumers;
                    n_skipped += skip ? 1u : 0u;
                }
            }
            const int n_copy = skip || empty ? 0 : n_ops;
            if (lane == 0) {
                StageMeta mt;
                mt.cx = kFloorMagicBits + bx0; mt.cy = kFloorMagicBits + by0;
                mt.rows2 = rows - 2;
                mt.sel = bw | (mode << 8) | ((mode == 0 && pc.fast != 0.0f ? (1 << k) : kSelSlow) << 16) | ((bx0 - bxs) << 10);
                if (kSkip && empty) mt.sel |= kSelEmpty;
                if constexpr (kReverse) {   // backward: a footprint too magnified for the int32 gradient box (BwdRing::kMagLimit)
                    const int ext_x = min(px0 + kTileW - 1, p.W - 1) - px0, ext_y = min(py0 + kTileH - 1, p.H - 1) - py0;
                    if (Ring::kMagLimit * (xmax - xmin - 1) < ext_x || Ring::kMagLimit * (ymax - ymin - 1) < ext_y) mt.sel &= 0xffff;
                }
                s_meta[s] = mt;
                // bytes the copies of this stage will deliver (a box counts whole, zero-filled parts included)
                const uint32_t tx = (uint32_t)((kFact ? kMaxBH : rows) * sw * (int)(4 * sizeof(E)));
                if (n_copy > 0 || kTBytes) mbar_arrive_expect_tx(&s_full[s], (n_copy > 0 ? tx : 0u) + kTBytes);
                else mbar_arrive(&s_full[s]);
                if (kReverse)   // the tile's saved transmittance for this plane rides in the same stage
                    tma_load_3d(s_buf + (size_t)s * kStride + kStageFloats, &maps.t, &s_full[s], px0, py0, v * N + i);
            }
            __syncwarp();
            // Few, tall copies.  UTMALDG takes uniform operands, so the lanes of a warp issue their copies ONE AFTER ANOTHER: with a
            // 4-row copy per lane (9-11 per stage, twice that for the factored MPI) the producer was the bottleneck of its own ring.
            if (n_copy > 0) {
                E* stage = s_buf + (size_t)s * kStride;
                if constexpr (kFact) {
                    // factored MPI: the colour box [row][3][bw] (shared image, or the last plane's own) starts the stage, as two or
                    // three copies that tile the ring's box height; the alpha box [row][bw] follows after 3/4 of the stage, as one copy
                    // of the full height.  Rows beyond the footprint are fetched and never read: the colour image is shared by all
                    // planes and comes from L2, alpha is a quarter of the bytes.
                    constexpr int kCR = Ring::kColourCopyRows;      // (a copy's destination must be 128-byte aligned, see the rings)
                    static_assert(kMaxBH % kCR == 0, "colour copies tile the box");
                    const CUtensorMap* cmap = (p.bg_rgb && i == N - 1) ? &maps.bg[k] : &maps.rgb[k];
                    if (lane < kMaxBH / kCR) tma_load_4d(stage + (size_t)lane * kCR * 3 * sw, cmap, &s_full[s], bxs, 0, by0 + lane * kCR, m);
                    if (lane == 31) tma_load_3d(stage + (kStageFloats / 4) * 3, &maps.a[k], &s_full[s], bxs, by0, m * N + i);
                } else if (!Ring::kBinaryCopies) {
                    // expanded MPI, backward: one 4-row copy per lane (measured: taller copies make its 2-stage ring 0.5 % slower)
                    if (lane < n_ops)
                        tma_load_4d(stage + (size_t)lane * kRowsPerOp * 4 * sw, &maps.m[k], &s_full[s], bxs, 0, by0 + lane * kRowsPerOp, m * N + i);
                } else if (lane < 4) {
                    // expanded MPI, forward (HBM-bound: no over-fetch): the n_ops 4-row chunks go out as the binary digits of n_ops,
                    // one copy of 32, 16, 8 and 4 rows each where the digit is set -- at most three copies for up to 44 rows (-1.1 %)
                    int before;
                    const int h = binary_copy_of_lane(n_ops, lane, before);
                    if (h) {
                        const CUtensorMap* mp = h == 8 ? &maps.m32[k] : h == 4 ? &maps.m16[k] : h == 2 ? &maps.m8[k] : &maps.m[k];
                        tma_load_4d(stage + (size_t)before * kRowsPerOp * 4 * sw, mp, &s_full[s], bxs, 0, by0 + before * kRowsPerOp, m * N + i);
                    }
                }
            }
        }
    }
    if constexpr (kES) {
        if (lane == 0 && n_skipped) atomicAdd(&g_early_stop_skipped, (unsigned long long)n_skipped);
    }
    if constexpr (kSkip) {
        if (lane == 0 && n_empty) atomicAdd(occ.skipped, (unsigned long long)n_empty);
    }
}

// 4x4 transpose inside every quad of lanes (4 q .. 4 q + 3): on entry lane k of a quad holds a[c] = M[k][c], on return
// a[t] = M[t][k].  Two butterfly steps, four shuffles.
__device__ __forceinline__ void quad_transpose(float (&a)[4], int lane) {
    const bool hi2 = (lane & 2) != 0, hi1 = (lane & 1) != 0;
    {   // exchange 2x2 blocks with lane ^ 2
        const float s0 = hi2 ? a[0] : a[2], s1 = hi2 ? a[1] : a[3];
        const float r0 = __shfl_xor_sync(0xffffffffu, s0, 2), r1 = __shfl_xor_sync(0xffffffffu, s1, 2);
        if (hi2) { a[0] = r0; a[1] = r1; } else { a[2] = r0; a[3] = r1; }
    }
    {   // exchange inside the 2x2 blocks with lane ^ 1
        const float s0 = hi1 ? a[0] : a[1], s1 = hi1 ? a[2] : a[3];
        const float r0 = __shfl_xor_sync(0xffffffffu, s0, 1), r1 = __shfl_xor_sync(0xffffffffu, s1, 1);
        if (hi1) { a[0] = r0; a[2] = r1; } else { a[1] = r0; a[3] = r1; }
    }
}

// Epilogue of one consumer warp, one pixel set at a time: o = (R, G, B, depth) of pixel (pxb + lane, py) of view v; all 32 lanes
// call this (the quad transpose shuffles).  Destinations:
//   * float4 stores after a quad transpose (lane k of a quad ends up with channel k of four consecutive x): 4 x STG.128 per
//     thread and tile instead of 16 x STG.32 -- and 4 per peer in the fused all-gather, or 4 in total through a multicast address;
//   * store_pixel for odd widths / unaligned outputs and for the uint8 video frames (render_video.py:118-126).
// (Collecting the four pixel sets in a [4][4] array first costs the plane loop 8 instructions per iteration through register
// pressure -- measured: -5 % frames/s -- so each set is stored as soon as it is formed.)
__device__ __forceinline__ void store_tile_pixels(const RenderParams& p, int v, size_t img, int pxb, int py, int lane, float (&o)[4]) {
    if (p.options & kOptVec4Stores) {      // (never set together with the video outputs)
        quad_transpose(o, lane);               // lane k of a quad now holds channel k of four consecutive x
        const int k = lane & 3, px = pxb + 4 * (lane >> 2);
        if (px >= p.W || py >= p.H) return;     // W % 4 == 0: a quad is inside or outside as a whole
        const float4 val = make_float4(o[0], o[1], o[2], o[3]);
        const size_t pix = (size_t)py * p.W + px;
        if (p.n_peers > 0) {
            const size_t fo = ((size_t)(p.frame_offset + v) * 4 + k) * img + pix;
            for (int r = 0; r < p.n_peers; ++r) *reinterpret_cast<float4*>(p.peer_frames[r] + fo) = val;
        } else {
            float* dst = k < 3 ? p.color + ((size_t)v * 3 + k) * img + pix : p.depth + (size_t)v * img + pix;
            *reinterpret_cast<float4*>(dst) = val;
        }
        return;
    }
    const int px = pxb + lane;
    if (px >= p.W || py >= p.H) return;
    store_pixel(p, v, img, (size_t)py * p.W + px, o[0], o[1], o[2], o[3]);
}

// Body of the staged forward kernels.  kES: early stop (kKeyES; s_stop is its stop-word ring, see kStopSlots).
// E: the MPI's element type (__half: GMPI_MPI_F16, the ring's boxes are fp16, each stage half the bytes).
// kSkip: empty-space skipping against `occ` (mpi_fwd_skip_kernel; forward only).
template <bool kAlignCorners, bool kEmitT, bool kFactored, bool kES, class E = float, bool kSkip = false>
__device__ __forceinline__ void fwd_staged_body(const RenderParams& p, const TmaMaps& maps, const int tiles_x, const int ring_stages,
                                                uint32_t* s_stop, OccMap occ = OccMap{}) {
    extern __shared__ __align__(1024) unsigned char smem_raw[];
    E* s_buf = reinterpret_cast<E*>(smem_raw);   // the ring starts the dynamic segment (1024-byte aligned)
    using Ring = FwdRing<kFactored, E>;
    static_assert(!(kFactored && std::is_same<E, uint8_t>::value), "uint8 MPIs are expanded");
    constexpr int kStages = Ring::kRingStages;              // ring stages allocated; the expanded MPI uses ring_stages of them
    const int n_stages = kFactored ? kStages : ring_stages;
    constexpr int kRingFloats = Ring::kPlaneFloats;         // floats per ring stage
    constexpr int kAOff = kFactored ? 3 * (kRingFloats / 4) : 0;      // factored: alpha box behind the colour box
    PlaneConst* s_pc = reinterpret_cast<PlaneConst*>(smem_raw + (size_t)n_stages * kRingFloats * sizeof(E));   // [N] of the current view
    __shared__ StageMeta s_meta[kStages];
    __shared__ __align__(8) uint64_t s_full[kStages], s_empty[kStages];
    __shared__ TileWalk s_walk;

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    if (threadIdx.x == 0) {
        s_walk.init(tiles_x, p.H, p.V, (int)blockIdx.x, (int)gridDim.x, kTileH, p.view_group);
        for (int s = 0; s < n_stages; ++s) {
            mbar_init(&s_full[s], 1);
            mbar_init(&s_empty[s], kConsWarps);
        }
        fence_mbar_init();
    }
    __syncthreads();

    const int Ht = p.Ht, Wt = p.Wt, N = p.N;
    const float fWt = (float)Wt, fHt = (float)Ht;
    float hsx = 0.5f * (float)(Wt - 1), hsy = 0.5f * (float)(Ht - 1);
    // Opaque to the optimiser: otherwise ptxas, short of registers, re-derives these two constants from the kernel parameters in
    // EVERY plane iteration (2 x LDCU + UIADD3 + I2FP + FMUL, the I2FP on the XU pipe behind the tap loads' MIO queue) -- seen
    // in the round-2 profile after unrelated prologue/epilogue changes: +3 % kernel time.
    asm volatile("" : "+f"(hsx), "+f"(hsy));
    int lane_ = lane;
    asm volatile("" : "+r"(lane_));     // likewise: no S2R + LOP3 per plane for the `lane == 0` of the arrive
    const size_t img = (size_t)p.H * p.W;

    if (warp == kConsWarps) {
        staged_producer<kAlignCorners, Ring, kFactored, kES, E, kSkip>(p, maps, s_buf, s_meta, s_full, s_empty, &s_walk, lane, n_stages,
                                                                        s_stop, occ);
    } else {
        // ================================ consumer warps ================================
        // warp w owns rows kPairs*w .. kPairs*w + kPairs-1 of the tile; a lane owns x = lane and lane+32 on each of them
        const bool check_last = (p.options & GMPI_CHECK_LAST_PLANE) != 0;
        const bool minus1_1 = (p.options & GMPI_COLOR_MINUS1_1) != 0;
        const float tau = kES ? p.early_stop : 0.0f;
        int c_stage = 0;            // ring position of this warp: stage index and mbarrier phase parity
        uint32_t c_phase = 0;
        uint32_t flag = 0;
        const size_t tex = (size_t)Ht * Wt;
        int v_table = -1;
        TileXY txy;
        for (int j = 0; s_walk.at(j, txy); ++j) {
            const int v = txy.v, px0 = txy.px0, py0 = txy.py0;
            const int m = __ldg(p.view2mpi + v);
            float ev[3], zd[3];
            load_eye_z(p, v, ev, zd);
            if (v != v_table) {          // (view, plane) constants, once per view and CTA
                consumer_bar_sync<kConsThreads>();     // everyone is done with the previous view's table
                // mpi.py:70 compares the distance of every plane the call renders (the MPIs of its views, not all p.M) with view 0's eye
                const float eye0_z = __ldg(p.eye0 + 2);
                for (int i = threadIdx.x; i < N; i += kConsThreads) {
                    const float* dp = p.dhw + ((size_t)m * N + i) * 3;
                    s_pc[i] = make_plane_const(dp, ev[2]);
                    if (!(__ldg(dp) >= eye0_z)) flag |= GMPI_FLAG_PLANE_BEHIND_EYE;
                }
                consumer_bar_sync<kConsThreads>();
                v_table = v;
            }
            if (py0 + kPairs * warp >= p.H) {      // warp-uniform: no row of this warp is inside the image
                consumer_idle_tile(s_full, s_empty, N, n_stages, lane, c_stage, c_phase);
                continue;
            }
            RayConst rc[kPix];   // scalar copies, only for the generic (rare) body and the epilogue
            RayPairs rp;
            bool rays_fast = (in_safe_range(ev[0]) || ev[0] == 0.0f) && (in_safe_range(ev[1]) || ev[1] == 0.0f);
#pragma unroll
            for (int q = 0; q < kPix; ++q) {
                const int px = min(px0 + lane + 32 * (q & 1), p.W - 1), py = min(py0 + kPairs * warp + (q >> 1), p.H - 1);
                float qx, qy, qz;
                load_ray(p, v, px, py, img, qx, qy, qz);
                rc[q] = make_ray_const(qx, qy, qz, ev, zd);
                rays_fast = rays_fast && rc[q].fast && fabsf(rc[q].rx2) <= 0x1p40f && fabsf(rc[q].ry2) <= 0x1p40f;
            }
            pack_ray_pairs(rc, rp);
            const f2 ex2 = splat(rc[0].ex2), ey2 = splat(rc[0].ey2), hsx2 = splat(hsx), hsy2 = splat(hsy);
            // warp-uniform: every ray of this warp is in the range where the reciprocal+FMA division is exact and no
            // coordinate can be NaN, so the per-plane body needs no per-pixel range checks
            const bool warp_fast = __all_sync(0xffffffffu, rays_fast);
            f2 T[kPairs], cr[kPairs], cg[kPairs], cb[kPairs], cws[kPairs];
#pragma unroll
            for (int P = 0; P < kPairs; ++P) { T[P] = splat(1.f); cr[P] = cg[P] = cb[P] = cws[P] = splat(0.f); }
            PlaneConst pc_next = s_pc[0];
            bool warp_stopped = false;     // kES: every pixel of this warp has stopped (warp-uniform)
            uint32_t* const stop_word = kES ? s_stop + (j & (kStopSlots - 1)) : nullptr;
            for (int i = 0; i < N; ++i) {
                const int s = c_stage;
                const uint32_t ph = c_phase;
                if (++c_stage == n_stages) { c_stage = 0; c_phase ^= 1u; }
                const PlaneConst pcc = pc_next;            // loaded one plane ahead: no shared-memory latency in front of the
                pc_next = s_pc[min(i + 1, N - 1)];         // coordinate chain (+1.3 %)
                CoordPairs cc;
                // Coordinates before the wait.  (Computing plane i+1's coordinates in the shadow of plane i's tap loads was
                // measured twice: -3 to -4 %; warps in their arithmetic phase leave the shared-memory pipe to the others.)
                if (warp_fast && !warp_stopped) coords_pairs<kAlignCorners>(pcc, rp, ex2, ey2, hsx2, hsy2, fWt, fHt, cc);
                if (kEmitT) {              // training: save T_i (before plane i) for the backward sweep, [V,N,H,W]
                    float* ts = p.transmittance + ((size_t)v * N + i) * img;
#pragma unroll
                    for (int q = 0; q < kPix; ++q) {
                        const int px = px0 + lane + 32 * (q & 1), py = py0 + kPairs * warp + (q >> 1);
                        if (px < p.W && py < p.H) ts[(size_t)py * p.W + px] = (q & 1) ? T[q >> 1].y : T[q >> 1].x;
                    }
                }
                mbar_wait(&s_full[s], ph);
                const StageMeta mt = s_meta[s];
                // the fp32 box's origin in the stage
                const E* sb = s_buf + s * kRingFloats + ((mt.sel >> 10) & ElemTraits<E>::kOriginMask);
                const int sel = mt.sel;                  // warp-uniform; the producer already folded mode and plane range in
                bool done = warp_stopped;                // a stopped warp only waits on and releases the stage
                if (warp_fast && !done) {
                    if (kSkip && (sel & kSelEmpty)) {    // empty box, not loaded: done when every tap of the warp falls in it
                        done = box_vote(mt.cx, mt.cy, (sel & 0xff) - 2, mt.rows2, cc);
                    } else if (Ring::kWideFact) {        // factored: two widths, both with bank-aligned row pitches
                        if (sel & (1 << 20)) done = sample_pairs<kWideBW, kAOff, kES, E>(sb, mt.cx, mt.cy, mt.rows2, cc, T, cr, cg, cb, cws, tau);
                        else if (sel & (1 << 17)) done = sample_pairs<64, kAOff, kES, E>(sb, mt.cx, mt.cy, mt.rows2, cc, T, cr, cg, cb, cws, tau);
                    } else {                             // most frequent classes first (FFHQ poses: 72 > 64 > 80 >> 56, 88)
                        if (sel & (1 << 18)) done = sample_pairs<72, kAOff, kES, E>(sb, mt.cx, mt.cy, mt.rows2, cc, T, cr, cg, cb, cws, tau);
                        else if (sel & (1 << 17)) done = sample_pairs<64, kAOff, kES, E>(sb, mt.cx, mt.cy, mt.rows2, cc, T, cr, cg, cb, cws, tau);
                        else if (sel & (1 << 19)) done = sample_pairs<80, kAOff, kES, E>(sb, mt.cx, mt.cy, mt.rows2, cc, T, cr, cg, cb, cws, tau);
                        else if (sel & (1 << 16)) done = sample_pairs<56, kAOff, kES, E>(sb, mt.cx, mt.cy, mt.rows2, cc, T, cr, cg, cb, cws, tau);
                        else if (sel & (1 << 20)) done = sample_pairs<88, kAOff, kES, E>(sb, mt.cx, mt.cy, mt.rows2, cc, T, cr, cg, cb, cws, tau);
                    }
                }
                if (!done) {
                    // ---- generic body: per-pixel range / box checks, direct sampling when not staged ----
                    const int bw = mt.sel & 0xff, mode = (mt.sel >> 8) & 3, bws = ElemTraits<E>::staged_width(bw, false), bw4 = 4 * bws;
                    const float fbw2 = (float)(bw - 2), fbh2 = (float)mt.rows2;
                    const float fbx0 = (float)(mt.cx - kFloorMagicBits), fby0 = (float)(mt.cy - kFloorMagicBits);
                    const E* plane = kFactored ? nullptr : reinterpret_cast<const E*>(p.rgba) + ((size_t)m * N + i) * 4 * tex;
                    float* Ts = reinterpret_cast<float*>(T);
                    float* crs = reinterpret_cast<float*>(cr);
                    float* cgs = reinterpret_cast<float*>(cg);
                    float* cbs = reinterpret_cast<float*>(cb);
                    float* cwss = reinterpret_cast<float*>(cws);
#pragma unroll
                    for (int q = 0; q < kPix; ++q) {
                        if (kES && fabsf(Ts[q]) <= tau) continue;   // stopped pixel: adds nothing
                        RayConst rg = rc[q];
                        rg.fast = false;            // rare path: plain IEEE divisions, no per-plane range checks in the hot loop
                        const TexCoord tc = plane_coord<kAlignCorners>(pcc, rg, hsx, hsy, fWt, fHt);
                        const float fx = floorf(tc.ix), fy = floorf(tc.iy);
                        const float rxx = fx - fbx0, ryy = fy - fby0;
                        float r, g, b, a;
                        if (kSkip && (mt.sel & kSelEmpty) && rxx >= 0.0f && rxx <= fbw2 && ryy >= 0.0f && ryy <= fbh2) {
                            continue;   // taps in the empty box: contributes exactly nothing
                        }
                        if (!kFactored && mode == 0 && rxx >= 0.0f && rxx <= fbw2 && ryy >= 0.0f && ryy <= fbh2) {
                            const float wx1 = tc.ix - fx, wy1 = tc.iy - fy;
                            const float wx0 = 1.0f - wx1, wy0 = 1.0f - wy1;
                            const float w00 = wx0 * wy0, w01 = wx1 * wy0, w10 = wx0 * wy1, w11 = wx1 * wy1;
                            const E* t0 = sb + ((int)ryy * bw4 + (int)rxx);
                            const E* t1 = t0 + bw4;
                            r = fmaf(to_f32(t1[1]), w11, fmaf(to_f32(t1[0]), w10, fmaf(to_f32(t0[1]), w01, to_f32(t0[0]) * w00)));
                            g = fmaf(to_f32(t1[bws + 1]), w11, fmaf(to_f32(t1[bws]), w10, fmaf(to_f32(t0[bws + 1]), w01, to_f32(t0[bws]) * w00)));
                            b = fmaf(to_f32(t1[2 * bws + 1]), w11,
                                     fmaf(to_f32(t1[2 * bws]), w10, fmaf(to_f32(t0[2 * bws + 1]), w01, to_f32(t0[2 * bws]) * w00)));
                            a = fmaf(to_f32(t1[3 * bws + 1]), w11,
                                     fmaf(to_f32(t1[3 * bws]), w10, fmaf(to_f32(t0[3 * bws + 1]), w01, to_f32(t0[3 * bws]) * w00)));
                        } else if (coord_hits(tc.ix, tc.iy, fWt, fHt)) {   // mode 1 ("nothing under the tile") is only the
                            // producer's corner-ray estimate: every pixel is still tested on its own
                            const float4 sv = sample_plane_any<kFactored, E>(p, plane, m, i, tex, tc.ix, tc.iy);
                            r = sv.x; g = sv.y; b = sv.z; a = sv.w;
                        } else {
                            continue;   // no texel under this ray on this plane: contributes exactly nothing
                        }
                        const float w = a * Ts[q];
                        crs[q] = fmaf(w, r, crs[q]);
                        cgs[q] = fmaf(w, g, cgs[q]);
                        cbs[q] = fmaf(w, b, cbs[q]);
                        cwss[q] = fmaf(w, tc.scale, cwss[q]);
                        Ts[q] -= w;
                    }
                }
                if constexpr (kES) {
                    if (!warp_stopped) {           // one vote per plane; the bit is published by the arrive below
                        bool st = true;
#pragma unroll
                        for (int P = 0; P < kPairs; ++P) st = st && fabsf(T[P].x) <= tau && fabsf(T[P].y) <= tau;
                        warp_stopped = __all_sync(0xffffffffu, st);
                        if (warp_stopped && i + 1 < N && lane_ == 0) atomicOr(stop_word, 1u << warp);
                    }
                }
                __syncwarp();
                mbar_arrive_if(&s_empty[s], lane_ == 0);    // predicated, no branch
            }
            if (check_last) {     // assert_not_out_of_last_plane, mpi.py:103-109 (once per tile)
                const PlaneConst pcl = s_pc[N - 1];
#pragma unroll
                for (int q = 0; q < kPix; ++q) {
                    RayConst rg = rc[q];
                    rg.fast = false;
                    const TexCoord tc = plane_coord<kAlignCorners>(pcl, rg, hsx, hsy, fWt, fHt);
                    if (!(tc.u >= -1.0f && tc.u <= 1.0f && tc.v >= -1.0f && tc.v <= 1.0f)) flag |= GMPI_FLAG_LAST_PLANE_OOB;
                }
            }
            // ---- epilogue: the warp's 2 rows x 64 pixels, (R, G, B, depth) per pixel, one pixel set at a time ----
#pragma unroll
            for (int q = 0; q < kPix; ++q) {
                float o[4];
                o[0] = (q & 1) ? cr[q >> 1].y : cr[q >> 1].x; o[1] = (q & 1) ? cg[q >> 1].y : cg[q >> 1].x;
                o[2] = (q & 1) ? cb[q >> 1].y : cb[q >> 1].x;
                o[3] = ((q & 1) ? cws[q >> 1].y : cws[q >> 1].x) * rc[q].dz;
                if (minus1_1) {
                    o[0] = fmaf(2.0f, o[0], -1.0f); o[1] = fmaf(2.0f, o[1], -1.0f); o[2] = fmaf(2.0f, o[2], -1.0f);
                }
                store_tile_pixels(p, v, img, px0 + 32 * (q & 1), py0 + kPairs * warp + (q >> 1), lane, o);
            }
        }
        if (flag) atomicOr(p.flags, flag);
    }
}

// The staged forward kernels by key (KeyTraits), without and with empty-space skipping against `occ` (two templates: the skipping
// kernels take one more parameter).  An early-stop kernel declares its stop-word ring in kernel scope, ahead of the body's shared
// variables, where the shared-memory offsets in its machine code come from.
template <uint32_t K>
__global__ void __launch_bounds__(kStagedThreads, 1)
mpi_fwd_staged_kernel(const RenderParams p, const __grid_constant__ TmaMaps maps, const int tiles_x, const int tiles_y,
                      const int ring_stages) {
    using T = KeyTraits<K>;
    static_assert((K & (kKeyStaged | kKeyBwd | kKeySkip)) == kKeyStaged, "a staged forward key without skipping");
    if constexpr (T::kES) {
        __shared__ uint32_t s_stop[kStopSlots];
        fwd_staged_body<T::kAlignCorners, T::kEmitT, T::kFactored, true, typename T::Elem>(p, maps, tiles_x, ring_stages, s_stop);
    } else {
        fwd_staged_body<T::kAlignCorners, T::kEmitT, T::kFactored, false, typename T::Elem>(p, maps, tiles_x, ring_stages, nullptr);
    }
}

template <uint32_t K>
__global__ void __launch_bounds__(kStagedThreads, 1)
mpi_fwd_skip_kernel(const RenderParams p, const __grid_constant__ TmaMaps maps, const int tiles_x, const int tiles_y,
                    const int ring_stages, const OccMap occ) {
    using T = KeyTraits<K>;
    static_assert((K & (kKeyStaged | kKeyBwd | kKeySkip | kKeyEmit)) == (kKeyStaged | kKeySkip), "a skipping forward key");
    if constexpr (T::kES) {
        __shared__ uint32_t s_stop[kStopSlots];
        fwd_staged_body<T::kAlignCorners, false, T::kFactored, true, typename T::Elem, true>(p, maps, tiles_x, ring_stages, s_stop, occ);
    } else {
        fwd_staged_body<T::kAlignCorners, false, T::kFactored, false, typename T::Elem, true>(p, maps, tiles_x, ring_stages, nullptr, occ);
    }
}

}  // namespace gmpi
