// MPI over-composite renderer for H100 (sm_90a): the C ABI (include/gmpi_mpi_render.h) and the table of this file's render kernels.
//
// Replaces gmpi/core/mpi.py MPI.forward (:308-436) + homography (:26-153) and their autograd.  The kernels live beside their
// siblings: the staged forward (mpi_fwd_staged.cuh), the direct forward and backward (mpi_fwd_direct.cuh, mpi_bwd_direct.cuh), the
// box backward and the deterministic backward's passes (mpi_bwd_box.cuh), the range check (mpi_range_check.cuh), the LightRenderer
// kernels (mpi_light.cuh) and the test hooks' kernels (mpi_debug.cuh).  Every kernel is launched through launch_args.
// DESIGN.md describes the data layout, each kernel and its roofline.
#include <cuda_runtime.h>
#include <stdarg.h>
#include <stdint.h>
#include <math.h>
#include <stdio.h>
#include <string.h>

#include <algorithm>
#include <atomic>
#include <iterator>
#include <mutex>
#include <tuple>
#include <type_traits>
#include <utility>

#include "../../include/gmpi_mpi_render.h"
#include "mpi_common.cuh"
#include "mpi_fwd_staged.cuh"
#include "mpi_bwd_box.cuh"
#include "mpi_light.cuh"
#include "mpi_fwd_direct.cuh"
#include "mpi_bwd_direct.cuh"
#include "mpi_range_check.cuh"
#include "mpi_debug.cuh"
#include "mpi_kernel_keys.cuh"

namespace gmpi {

// ------------------------------------------------------------------------------------------
// error plumbing
// ------------------------------------------------------------------------------------------
static thread_local char g_err[512] = "";

static int fail(int code, const char* fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
    return code;
}

#define GMPI_CUDA_OK(expr)                                                                        \
    do {                                                                                          \
        cudaError_t _e = (expr);                                                                  \
        if (_e != cudaSuccess)                                                                    \
            return fail(GMPI_ERR_CUDA, "%s failed: %s (%s:%d)", #expr, cudaGetErrorString(_e),    \
                        __FILE__, __LINE__);                                                      \
    } while (0)

}  // namespace gmpi

using namespace gmpi;

static std::atomic<int> g_fwd_variant{0};   // 0 auto, 1 direct, 2 staged (test hook; relaxed atomic: any thread may set it)
static std::atomic<int> g_fwd_stages{0};    // expanded staged forward's ring depth: 0 auto (fwd_ring_stages), 2 or 3 (test hook)

// An MPI is factored (rgb + alpha [+ bg_rgb]) or expanded (rgba).
static bool factored(const RenderParams& p) { return p.alpha != nullptr; }

// The sizes of the MPIs, and with `views` those of the views too.  `texels`: the texels of one channel must also stay below 2^31.
static int check_sizes(const RenderParams& p, bool views, bool texels) {
    if (views && (p.M < 1 || p.V < 0 || p.N < 1 || p.Ht < 1 || p.Wt < 1 || p.H < 1 || p.W < 1))
        return fail(GMPI_ERR_INVALID_ARGUMENT, "bad sizes M=%d V=%d N=%d Ht=%d Wt=%d H=%d W=%d", p.M, p.V, p.N, p.Ht, p.Wt, p.H, p.W);
    if (p.M < 1 || p.N < 1 || p.Ht < 1 || p.Wt < 1)
        return fail(GMPI_ERR_INVALID_ARGUMENT, "bad sizes M=%d N=%d Ht=%d Wt=%d", p.M, p.N, p.Ht, p.Wt);
    if (texels && (size_t)p.Ht * p.Wt > (size_t)0x7fffffff)
        return fail(GMPI_ERR_UNSUPPORTED, "texture of %dx%d texels exceeds 2^31 elements per channel", p.Ht, p.Wt);
    return GMPI_OK;
}

// The forward-only options.  A backward call refuses them, and so does a forward that saves the transmittance for one (the
// training forward).  Those refusals come from this table, in its order; `why`: why the backward cannot take the option.
struct ForwardOnly { uint32_t bit; const char *name, *why; };
static const ForwardOnly kForwardOnly[] = {
    {GMPI_MPI_F16, "GMPI_MPI_F16", "the backward reads and writes fp32 MPIs"},
    {GMPI_MPI_U8, "GMPI_MPI_U8", "the backward reads and writes fp32 MPIs"},
    {GMPI_EARLY_STOP, "GMPI_EARLY_STOP", "the backward needs every plane's samples"},
};

// The calls check_call knows.  A classic entry point fills a descriptor and is checked as the call it corresponds to.
enum CallKind {
    kFwdCall,         // gmpi_mpi_render_fwd_ex; the classic fwd, fwd_train and fwd_gather
    kSkipCall,        // gmpi_mpi_render_fwd_skip_ex
    kHostCall,        // gmpi_mpi_render_host_ex (host buffers); the classic fwd_host
    kBwdCall,         // gmpi_mpi_render_bwd_ex and gmpi_mpi_render_bwd_deterministic_ex; the classic bwd and bwd_saved
    kBwdPlanCall,     // gmpi_mpi_render_bwd_plan_ex: kBwdCall's checks less those that a pointer is set (it reads pointer values only)
    kOccQueryCall,    // gmpi_mpi_occupancy_bytes
    kOccBuildCall,    // gmpi_mpi_build_occupancy
    kScratchCall,     // gmpi_mpi_render_bwd_deterministic_scratch_bytes
};

struct Call {
    CallKind kind;
    bool classic = false;                     // from a classic entry point
    const char* classic_refusal = nullptr;    // that entry point's own refusal of its arguments (nullptr: none)
    const void* occ = nullptr; size_t occ_bytes = 0;    // the occupancy map of kSkipCall and kOccBuildCall
};

// Occupancy map: M*N planes of occ_rows(Ht) block rows of occ_words(Wt) words.
static size_t occ_map_bytes(const RenderParams& p) { return (size_t)p.M * p.N * occ_rows(p.Ht) * occ_words(p.Wt) * sizeof(uint32_t); }

static int check_occ_map(const RenderParams& p, const Call& c) {
    if (!c.occ) return fail(GMPI_ERR_INVALID_ARGUMENT, "null occupancy map (gmpi_mpi_occupancy_bytes gives its size)");
    if ((uintptr_t)c.occ & 3) return fail(GMPI_ERR_INVALID_ARGUMENT, "the occupancy map must be 4-byte aligned");
    const size_t need = occ_map_bytes(p);
    if (c.occ_bytes < need)
        return fail(GMPI_ERR_INVALID_ARGUMENT, "occupancy map of %zu bytes is smaller than the %zu bytes of this MPI", c.occ_bytes, need);
    return GMPI_OK;
}

// Every check of a call's RenderParams, and of the occupancy map it reads.  The first refusal wins.
static int check_call(const RenderParams& p, const Call& c) {
    // A classic entry point takes no forward-only option.  Its MPI pointer is a float*, so fp16 and uint8 are refused first.  It has
    // no early_stop field, so GMPI_EARLY_STOP is refused where a descriptor's threshold is checked.
    for (const ForwardOnly& o : kForwardOnly)
        if (c.classic && (p.options & o.bit & (GMPI_MPI_F16 | GMPI_MPI_U8)))
            return fail(GMPI_ERR_UNSUPPORTED, "%s is accepted by the descriptor forward entry points only", o.name);
    if (c.classic_refusal) return fail(GMPI_ERR_INVALID_ARGUMENT, "%s", c.classic_refusal);
    // the uint8 MPI's own rules: not fp16 as well (here), and expanded only (after the backward's refusals)
    if ((p.options & GMPI_MPI_U8) && (p.options & GMPI_MPI_F16))
        return fail(GMPI_ERR_INVALID_ARGUMENT, "GMPI_MPI_U8 and GMPI_MPI_F16 are exclusive");
    // Of the forward-only options, the occupancy calls and the scratch query check GMPI_MPI_U8 alone: the scratch query returns a size
    // for GMPI_MPI_F16 and GMPI_EARLY_STOP, which the deterministic backward refuses.
    const bool occ = c.kind == kOccQueryCall || c.kind == kOccBuildCall, plan = c.kind == kBwdPlanCall,
               bwd = c.kind == kBwdCall || c.kind == kScratchCall || plan;
    const uint32_t opts = p.options & (occ || c.kind == kScratchCall ? GMPI_MPI_U8 : GMPI_MPI_F16 | GMPI_MPI_U8 | GMPI_EARLY_STOP);
    for (const ForwardOnly& o : kForwardOnly)
        if (bwd && (opts & o.bit)) return fail(GMPI_ERR_UNSUPPORTED, "%s is forward-only: %s", o.name, o.why);
    if ((opts & GMPI_MPI_U8) && (p.rgb || p.alpha || p.bg_rgb))
        return fail(GMPI_ERR_UNSUPPORTED, "GMPI_MPI_U8 takes an expanded MPI (rgba), not a factored one");
    for (const ForwardOnly& o : kForwardOnly)
        if ((opts & o.bit) && p.transmittance)
            return fail(GMPI_ERR_UNSUPPORTED, "%s cannot be combined with the training forward (transmittance)", o.name);
    if ((opts & GMPI_EARLY_STOP) && c.classic)
        return fail(GMPI_ERR_INVALID_ARGUMENT, "GMPI_EARLY_STOP needs a descriptor: the classic entry points have no early_stop field");
    if ((opts & GMPI_EARLY_STOP) && !(p.early_stop >= 0.0f && p.early_stop < 1.0f))
        return fail(GMPI_ERR_INVALID_ARGUMENT, "early_stop = %g must be in [0, 1) (gmpi_render_desc.early_stop)", (double)p.early_stop);
    if (c.kind == kScratchCall) return check_sizes(p, true, false);
    if (!plan && (factored(p) ? !p.rgb || p.rgba : !p.rgba || p.rgb))
        return fail(GMPI_ERR_INVALID_ARGUMENT, "null input pointer (MPI: pass rgba, or rgb + alpha)");
    if (occ) {
        if (int rc = check_sizes(p, false, true)) return rc;
        return c.kind == kOccBuildCall ? check_occ_map(p, c) : GMPI_OK;
    }
    if (!plan && (!p.view2mpi || !p.dhw)) return fail(GMPI_ERR_INVALID_ARGUMENT, "null input pointer");
    if (!plan && !p.cam && (!p.ray_dir || !p.eye || !p.z_dir))
        return fail(GMPI_ERR_INVALID_ARGUMENT, "null input pointer (camera: pass ray_dir + eye + z_dir, or cam)");
    if (int rc = check_sizes(p, true, true)) return rc;
    if (p.view_group < 0 || (p.view_group > 1 && p.V % p.view_group != 0))
        return fail(GMPI_ERR_INVALID_ARGUMENT, "view_group=%d does not divide V=%d", p.view_group, p.V);
    if (bwd) {
        if (p.cam) return fail(GMPI_ERR_UNSUPPORTED, "the backward needs the reference's ray tensors (cam is forward-only)");
        if (plan) return GMPI_OK;
        if (!p.g_color) return fail(GMPI_ERR_INVALID_ARGUMENT, "null gradient pointer");
        if (factored(p) ? (!p.g_rgb || !p.g_alpha || (p.bg_rgb && !p.g_bg_rgb) || p.g_rgba) : !p.g_rgba)
            return fail(GMPI_ERR_INVALID_ARGUMENT, "null gradient pointer (pass g_rgba, or g_rgb + g_alpha [+ g_bg_rgb])");
        return GMPI_OK;
    }
    if (c.kind == kSkipCall) {
        if (p.transmittance)
            return fail(GMPI_ERR_UNSUPPORTED, "empty-space skipping is forward-only: it cannot be combined with the training forward (transmittance)");
        if (int rc = check_occ_map(p, c)) return rc;
    }
    // the forward's outputs
    if (c.kind == kHostCall) {
        if (!p.flags || (!p.video_rgb && (!p.color || !p.depth))) return fail(GMPI_ERR_INVALID_ARGUMENT, "null output pointer");
        if (p.n_peers > 0 || p.transmittance) return fail(GMPI_ERR_UNSUPPORTED, "the host entry point renders to host buffers only");
    } else if (!p.flags) {
        return fail(GMPI_ERR_INVALID_ARGUMENT, "null flags pointer");
    }
    if (p.video_rgb) {
        if (p.n_peers > 0) return fail(GMPI_ERR_INVALID_ARGUMENT, "video outputs and peer frames are exclusive");
        if (p.video_depth && !(p.depth_range != 0.0f)) return fail(GMPI_ERR_INVALID_ARGUMENT, "depth_range must be non-zero");
    } else if (p.n_peers > 0) {
        if (!p.peer_frames || p.frame_offset < 0) return fail(GMPI_ERR_INVALID_ARGUMENT, "bad peer frame buffers");
    } else if (!p.color || !p.depth) {
        return fail(GMPI_ERR_INVALID_ARGUMENT, "null output pointer");
    }
    return GMPI_OK;
}

static bool aligned16(const void* a) { return ((uintptr_t)a & 15) == 0; }

// The element type E of a checked call's MPI: fp16 under GMPI_MPI_F16, uint8 under GMPI_MPI_U8 (exclusive, check_call), else fp32.
// Returns f(ElemTraits<E>{}).
template <class F>
static auto with_mpi_elem(uint32_t options, F&& f) {
    if (options & GMPI_MPI_U8) return f(ElemTraits<uint8_t>{});
    if (options & GMPI_MPI_F16) return f(ElemTraits<__half>{});
    return f(ElemTraits<float>{});
}

// The GMPI_WHY_* bits of every reason the TMA-staged forward is not launched for p (0 = staged): the one decision behind
// launch_fwd, launch_bwd and the plan queries.  The tensor maps need 16-byte row strides (Wt % ElemTraits<E>::kAlign == 0: 4 in
// fp32, 8 in fp16, 16 in uint8) and 16-byte aligned MPI bases (NULL counts as aligned); the plane-constant table holds
// kMaxPlanesStaged planes, and the M*N planes of all MPIs stay below 2^31; the persistent grid needs enough tiles.  Reads the sizes,
// the fp16 and uint8 bits, the MPI pointers and the variant override, nothing else: the early-stop and training instantiations get
// the plain forward's plan.
static uint32_t fwd_why(const RenderParams& p) {
    uint32_t w = 0;
    if (p.N > kMaxPlanesStaged || (size_t)p.M * p.N >= ((size_t)1 << 31)) w |= GMPI_WHY_MANY_PLANES;
    if (with_mpi_elem(p.options, [&](auto e) { return p.Wt % decltype(e)::kAlign; }) != 0) w |= GMPI_WHY_TEX_WIDTH;
    if (!(factored(p) ? aligned16(p.rgb) && aligned16(p.alpha) && aligned16(p.bg_rgb) : aligned16(p.rgba))) w |= GMPI_WHY_ALIGNMENT;
    const int forced = g_fwd_variant.load(std::memory_order_relaxed);
    if (forced == 1) w |= GMPI_WHY_FORCED;
    const long tiles = (long)((p.W + kTileW - 1) / kTileW) * ((p.H + kTileH - 1) / kTileH) * p.V;
    if (forced != 2 && tiles < 120) w |= GMPI_WHY_FEW_TILES;
    return w;
}

// Tensor maps of the MPI (expanded or factored) for the five box-width classes.  Returns 0 on success.
// box_h, colour_rows: the ring's box height and kColourCopyRows (factored: colour copies of colour_rows rows, one alpha copy of box_h).
// wide: the factored forward's ring (FwdRing<true, E>) -- slot 4 holds the kWideBW-wide boxes, slot 1 the 64-wide ones, the rest
// unused.  The maps are of the MPI's element type, with its staged box widths (ElemTraits).
static int encode_mpi_maps(TmaMaps& maps, const RenderParams& p, int box_h, int colour_rows, bool wide = false) {
    const MapElem el = with_mpi_elem(p.options, [](auto e) { return decltype(e)::kMap; });
    for (int k = 0; k < kNumMaps; ++k) {
        const int bw = with_mpi_elem(p.options, [&](auto e) { return decltype(e)::staged_width(class_width(k, wide), wide); });
        if (factored(p)) {
            if (encode_color_map(&maps.rgb[k], p.rgb, el, (uint64_t)p.M, p.Ht, p.Wt, bw, colour_rows) != 0) return -1;
            if (p.bg_rgb && encode_color_map(&maps.bg[k], p.bg_rgb, el, (uint64_t)p.M, p.Ht, p.Wt, bw, colour_rows) != 0) return -1;
            if (encode_slab_map(&maps.a[k], p.alpha, el, (uint64_t)p.M * p.N, p.Ht, p.Wt, bw, box_h, 1) != 0) return -1;
        } else {
            CUtensorMap* const by_rows[4] = {&maps.m[k], &maps.m8[k], &maps.m16[k], &maps.m32[k]};
            for (int b = 0; b < 4; ++b)
                if (encode_plane_map(by_rows[b], p.rgba, el, (uint64_t)p.M * p.N, p.Ht, p.Wt, bw, kRowsPerOp << b) != 0) return -1;
        }
    }
    return 0;
}

static int device_attr(cudaDeviceAttr attr, int* value) {
    int dev = 0;
    GMPI_CUDA_OK(cudaGetDevice(&dev));
    GMPI_CUDA_OK(cudaDeviceGetAttribute(value, attr, dev));
    return GMPI_OK;
}

// Ring depth of the expanded forward.  When every view has an MPI of its own that is larger than L2, each box streams from
// HBM, and a shallower ring is faster: 2 stages take 0.85x the time of 3 at 4 MPIs x 96 planes x 1024^2, 4 stages 1.10x.
// When the boxes come from L2 (views sharing an MPI, or an MPI that fits L2) 3 stages are faster (DESIGN.md section 4.1).
static int fwd_ring_stages(const RenderParams& p, int l2_bytes) {
    const bool shared_mpi = p.view_group > 1 || p.V > p.M;
    const bool fits_l2 = (double)p.N * p.Ht * p.Wt * 16.0 <= (double)l2_bytes;
    return shared_mpi || fits_l2 ? kStages : kStreamStages;
}

// The render kernels of this file.  This table is the first reference to each kernel template here, so its order is the order the
// kernels are instantiated in, and ptxas gives some kernels other machine code when that order changes (the expanded box
// backward's, when the four box kernels are listed by [align_corners][factored]).  Do not reorder it: the recorded SASS digests
// (tests/golden/sass_digests.json) check the machine code.
static const RenderKernel kRenderKernels[] = {
    {kKeyStaged, mpi_fwd_staged_kernel<kKeyStaged>},
    {kKeyStaged | kKeyFac, mpi_fwd_staged_kernel<kKeyStaged | kKeyFac>},
    {kKeyStaged | kKeyEmit, mpi_fwd_staged_kernel<kKeyStaged | kKeyEmit>},
    {kKeyStaged | kKeyEmit | kKeyFac, mpi_fwd_staged_kernel<kKeyStaged | kKeyEmit | kKeyFac>},
    {kKeyStaged | kKeyAC, mpi_fwd_staged_kernel<kKeyStaged | kKeyAC>},
    {kKeyStaged | kKeyAC | kKeyFac, mpi_fwd_staged_kernel<kKeyStaged | kKeyAC | kKeyFac>},
    {kKeyStaged | kKeyAC | kKeyEmit, mpi_fwd_staged_kernel<kKeyStaged | kKeyAC | kKeyEmit>},
    {kKeyStaged | kKeyAC | kKeyEmit | kKeyFac, mpi_fwd_staged_kernel<kKeyStaged | kKeyAC | kKeyEmit | kKeyFac>},
    {kKeyStaged | kKeyES, mpi_fwd_staged_kernel<kKeyStaged | kKeyES>},
    {kKeyStaged | kKeyES | kKeyFac, mpi_fwd_staged_kernel<kKeyStaged | kKeyES | kKeyFac>},
    {kKeyStaged | kKeyES | kKeyAC, mpi_fwd_staged_kernel<kKeyStaged | kKeyES | kKeyAC>},
    {kKeyStaged | kKeyES | kKeyAC | kKeyFac, mpi_fwd_staged_kernel<kKeyStaged | kKeyES | kKeyAC | kKeyFac>},
    {0, mpi_fwd_direct_kernel<0>},
    {kKeyAC, mpi_fwd_direct_kernel<kKeyAC>},
    {kKeyES, mpi_fwd_direct_kernel<kKeyES>},
    {kKeyES | kKeyAC, mpi_fwd_direct_kernel<kKeyES | kKeyAC>},
    {kKeyF16 | kKeyStaged, mpi_fwd_staged_kernel<kKeyF16 | kKeyStaged>},
    {kKeyF16 | kKeyStaged | kKeyFac, mpi_fwd_staged_kernel<kKeyF16 | kKeyStaged | kKeyFac>},
    {kKeyF16 | kKeyStaged | kKeyAC, mpi_fwd_staged_kernel<kKeyF16 | kKeyStaged | kKeyAC>},
    {kKeyF16 | kKeyStaged | kKeyAC | kKeyFac, mpi_fwd_staged_kernel<kKeyF16 | kKeyStaged | kKeyAC | kKeyFac>},
    {kKeyF16 | kKeyStaged | kKeyES, mpi_fwd_staged_kernel<kKeyF16 | kKeyStaged | kKeyES>},
    {kKeyF16 | kKeyStaged | kKeyES | kKeyFac, mpi_fwd_staged_kernel<kKeyF16 | kKeyStaged | kKeyES | kKeyFac>},
    {kKeyF16 | kKeyStaged | kKeyES | kKeyAC, mpi_fwd_staged_kernel<kKeyF16 | kKeyStaged | kKeyES | kKeyAC>},
    {kKeyF16 | kKeyStaged | kKeyES | kKeyAC | kKeyFac, mpi_fwd_staged_kernel<kKeyF16 | kKeyStaged | kKeyES | kKeyAC | kKeyFac>},
    {kKeyF16, mpi_fwd_direct_kernel<kKeyF16>},
    {kKeyF16 | kKeyAC, mpi_fwd_direct_kernel<kKeyF16 | kKeyAC>},
    {kKeyF16 | kKeyES, mpi_fwd_direct_kernel<kKeyF16 | kKeyES>},
    {kKeyF16 | kKeyES | kKeyAC, mpi_fwd_direct_kernel<kKeyF16 | kKeyES | kKeyAC>},
    {kKeyBwd | kKeyDet | kKeyAC, mpi_bwd_direct_det_kernel<kKeyBwd | kKeyDet | kKeyAC>},
    {kKeyBwd | kKeyDet, mpi_bwd_direct_det_kernel<kKeyBwd | kKeyDet>},
    {kKeyBwd | kKeyAC, mpi_bwd_direct_kernel<kKeyBwd | kKeyAC>},
    {kKeyBwd, mpi_bwd_direct_kernel<kKeyBwd>},
    {kKeyBwd | kKeyDet | kKeyStaged | kKeyAC | kKeyFac, mpi_bwd_box_det_kernel<kKeyBwd | kKeyDet | kKeyStaged | kKeyAC | kKeyFac>},
    {kKeyBwd | kKeyDet | kKeyStaged | kKeyFac, mpi_bwd_box_det_kernel<kKeyBwd | kKeyDet | kKeyStaged | kKeyFac>},
    {kKeyBwd | kKeyDet | kKeyStaged | kKeyAC, mpi_bwd_box_det_kernel<kKeyBwd | kKeyDet | kKeyStaged | kKeyAC>},
    {kKeyBwd | kKeyDet | kKeyStaged, mpi_bwd_box_det_kernel<kKeyBwd | kKeyDet | kKeyStaged>},
    {kKeyBwd | kKeyStaged | kKeyAC | kKeyFac, mpi_bwd_box_kernel<kKeyBwd | kKeyStaged | kKeyAC | kKeyFac>},
    {kKeyBwd | kKeyStaged | kKeyFac, mpi_bwd_box_kernel<kKeyBwd | kKeyStaged | kKeyFac>},
    {kKeyBwd | kKeyStaged | kKeyAC, mpi_bwd_box_kernel<kKeyBwd | kKeyStaged | kKeyAC>},
    {kKeyBwd | kKeyStaged, mpi_bwd_box_kernel<kKeyBwd | kKeyStaged>},
};

// mpi_render.cu has no skipping kernels, so no skip counter.
static cudaError_t render_stage_counters(unsigned long long** early_stop, unsigned long long** empty) {
    *empty = nullptr;
    return cudaGetSymbolAddress(reinterpret_cast<void**>(early_stop), g_early_stop_skipped);
}

const KernelUnit gmpi::render_unit = {std::begin(kRenderKernels), std::end(kRenderKernels), render_stage_counters};

// The translation unit that defines the kernel of `key`.
static const KernelUnit& key_unit(uint32_t key) {
    return (key & kKeyU8) ? u8_unit : (key & kKeySkip) ? skip_unit : render_unit;
}

// Every render kernel by its key.  A key without a kernel gives nullptr, which the launch refuses.
static const void* render_kernel(uint32_t key) {
    const KernelUnit& u = key_unit(key);
    const RenderKernel* k = std::find_if(u.begin, u.end, [key](const RenderKernel& r) { return r.key == key; });
    return k == u.end ? nullptr : k->kernel;
}

// Everything one render-kernel launch needs.  The arguments point into this object, so it is built in place and never copied.
struct Launch {
    uint32_t key = 0;                // the kernel's key (render_kernel)
    dim3 grid, block;
    size_t smem = 0;
    long tiles = 0;                  // the tiles of all views a persistent kernel walks (0: a direct kernel)
    RenderParams p;                  // the first argument of every render kernel
    TmaMaps maps;
    int ints[3] = {};                // a persistent kernel's tiles_x, tiles_y and ring stages; the direct backward's tile_w, tile_h
    OccMap om;
    DetAcc da;
    void* args[6] = {&p};
    int n_args = 1;
    // the set-up every render launch shares: the call's view-0 eye (the host entry point sets its own) and one view per group
    explicit Launch(const RenderParams& q) : p(q) {
        if (!p.eye0) p.eye0 = p.cam ? p.cam + 13 : p.eye;
        if (p.view_group < 1) p.view_group = 1;
    }
    Launch(const Launch&) = delete;
    void arg(void* a) { args[n_args++] = a; }
};

// Every kernel launch of the library: `args` holds the address of each of the kernel's arguments, in order.  Reports this launch's
// own error, not one the calling thread left pending, and lifts the kernel's dynamic shared-memory limit when smem exceeds 48 KB.
static int launch_args(const void* kernel, dim3 grid, dim3 block, size_t smem, cudaStream_t st, void** args) {
    if (smem > 48 * 1024) GMPI_CUDA_OK(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    cudaLaunchConfig_t cfg = {grid, block, smem, st, nullptr, 0};
    GMPI_CUDA_OK(cudaLaunchKernelExC(&cfg, kernel, args));
    return GMPI_OK;
}

// A launch of every kernel but the render kernels (whose arguments vary by key: Launch).  Each argument is converted to its
// parameter's type P, so the compiler checks the arguments against the kernel's parameter list.
template <class... P, class... A>
static int launch_kernel(void (*kernel)(P...), dim3 grid, dim3 block, size_t smem, cudaStream_t st, A&&... a) {
    static_assert(sizeof...(P) == sizeof...(A), "one argument per kernel parameter");
    std::tuple<P...> params(std::forward<A>(a)...);
    return std::apply([&](P&... x) {
        void* arg_addrs[] = {&x...};
        return launch_args(reinterpret_cast<const void*>(kernel), grid, block, smem, st, arg_addrs);
    }, params);
}

// The test hook gmpi_debug_last_render_key: per device, 1 + the key of the last render kernel launch() launched there (0: none yet).
constexpr int kMaxKeyDevices = 64;
static std::atomic<uint64_t> g_last_render_key[kMaxKeyDevices];

static int launch(Launch& l, cudaStream_t st) {
    if (int rc = launch_args(render_kernel(l.key), l.grid, l.block, l.smem, st, l.args)) return rc;
    int dev = 0;
    if (cudaGetDevice(&dev) == cudaSuccess && dev >= 0 && dev < kMaxKeyDevices)
        g_last_render_key[dev].store((uint64_t)l.key + 1, std::memory_order_relaxed);
    return GMPI_OK;
}

// The persistent grid of the staged forward and the box backward: tiles of kTileW x tile_h pixels in every view, at most one CTA
// per SM.  Also adds the arguments both kernels take after p: maps, tiles_x, tiles_y.
static int persistent_grid(Launch& l, int tile_h) {
    const RenderParams& p = l.p;
    int sms = 0;
    if (int rc = device_attr(cudaDevAttrMultiProcessorCount, &sms)) return rc;
    l.ints[0] = (p.W + kTileW - 1) / kTileW;
    l.ints[1] = (p.H + tile_h - 1) / tile_h;
    l.tiles = (long)l.ints[0] * l.ints[1] * p.V;
    l.grid = dim3((unsigned)(l.tiles < sms ? l.tiles : sms));
    l.arg(&l.maps);
    l.arg(&l.ints[0]);
    l.arg(&l.ints[1]);
    return GMPI_OK;
}

// Dynamic shared memory of the staged forward kernel of p: its ring (FwdRing of the kernel's kFactored and the MPI's element type;
// stages of them when expanded, kStages when factored) and the plane-constant table.
static size_t fwd_staged_smem(const RenderParams& p, int stages) {
    const size_t ring = with_mpi_elem(p.options, [&](auto e) {
        using E = typename decltype(e)::Elem;
        return factored(p) ? kStages * FwdRing<true, E>::kStageBytes : stages * FwdRing<false, E>::kStageBytes;
    });
    return ring + (size_t)kMaxPlanesStaged * 32;
}

// The stage counters of the test hooks gmpi_debug_fwd_early_stop_stats and gmpi_debug_fwd_skip_stats: on the device, the stages
// the last early-stop or skipping launch armed without copies (zeroed on its stream); here, the (tile, plane) stages it walked and
// the unit whose kernel it launched (KernelUnit::stage_counters).  The direct kernels count no stages: their counters read 0.
enum StageStats { kEarlyStopStats, kSkipStats };
static std::atomic<unsigned long long> g_stages_walked[2];
static std::atomic<const KernelUnit*> g_stages_unit[2] = {{&render_unit}, {&render_unit}};

// The device counter on the current device; nullptr: the unit has no such counter, which reads 0.
static int stage_counter(StageStats s, const KernelUnit& unit, unsigned long long** counter) {
    unsigned long long* c[2] = {nullptr, nullptr};
    GMPI_CUDA_OK(unit.stage_counters(&c[kEarlyStopStats], &c[kSkipStats]));
    *counter = c[s];
    return GMPI_OK;
}

static int reset_stage_stats(StageStats s, const KernelUnit& unit, unsigned long long walked, cudaStream_t st) {
    unsigned long long* counter = nullptr;
    if (int rc = stage_counter(s, unit, &counter)) return rc;
    if (counter) GMPI_CUDA_OK(cudaMemsetAsync(counter, 0, sizeof(unsigned long long), st));
    g_stages_walked[s].store(walked, std::memory_order_relaxed);
    g_stages_unit[s].store(&unit, std::memory_order_relaxed);
    return GMPI_OK;
}

static int read_stage_stats(StageStats s, unsigned long long* skipped, unsigned long long* walked) {
    if (!skipped || !walked) return fail(GMPI_ERR_INVALID_ARGUMENT, "null pointer");
    unsigned long long* counter = nullptr;
    if (int rc = stage_counter(s, *g_stages_unit[s].load(std::memory_order_relaxed), &counter)) return rc;
    GMPI_CUDA_OK(cudaDeviceSynchronize());
    *skipped = 0;
    if (counter) GMPI_CUDA_OK(cudaMemcpy(skipped, counter, sizeof(unsigned long long), cudaMemcpyDeviceToHost));
    *walked = g_stages_walked[s].load(std::memory_order_relaxed);
    return GMPI_OK;
}

// The forward kernel of a checked call with V > 0, with its launch.  occ: empty-space skipping against this map.  The staged
// kernel when fwd_why(p) == 0 and its tensor maps encode, else the direct kernel; a forced staged variant fails instead.
static int fwd_launch(Launch& l, const uint32_t* occ) {
    const RenderParams& p = l.p;
    const bool fac = factored(p);
    uint32_t key = ((p.options & GMPI_ALIGN_CORNERS) ? kKeyAC : 0) | ((p.options & GMPI_EARLY_STOP) ? kKeyES : 0) |
                   ((p.options & GMPI_MPI_F16) ? kKeyF16 : 0) | ((p.options & GMPI_MPI_U8) ? kKeyU8 : 0);
    int rc = GMPI_OK;
    if (fwd_why(p) == 0) {
        if (encode_mpi_maps(l.maps, p, kMaxBH, FwdRing<true, float>::kColourCopyRows, fac) == 0) {
            int l2 = 0;
            if ((rc = persistent_grid(l, kTileH)) != 0) return rc;
            if ((rc = device_attr(cudaDevAttrL2CacheSize, &l2)) != 0) return rc;
            const int forced_stages = g_fwd_stages.load(std::memory_order_relaxed);
            l.ints[2] = forced_stages ? forced_stages : fwd_ring_stages(p, l2);
            l.block = dim3(kStagedThreads);
            l.smem = fwd_staged_smem(p, l.ints[2]);
            l.arg(&l.ints[2]);
            key |= kKeyStaged | (fac ? kKeyFac : 0) | (occ ? kKeySkip : 0) | (p.transmittance ? kKeyEmit : 0);
            l.key = key;
            if (!occ) return GMPI_OK;
            l.om = OccMap{occ, occ_words(p.Wt), occ_rows(p.Ht), nullptr};
            l.arg(&l.om);
            return stage_counter(kSkipStats, key_unit(key), &l.om.skipped);
        }
        if (g_fwd_variant.load(std::memory_order_relaxed) == 2) return fail(GMPI_ERR_CUDA, "cuTensorMapEncodeTiled failed");
    }
    l.p.options &= ~kOptVec4Stores;      // the direct kernel stores pixel by pixel
    l.smem = sizeof(PlaneConst) * (size_t)p.N;
    if (l.smem > 200 * 1024) return fail(GMPI_ERR_UNSUPPORTED, "N=%d planes exceed the shared-memory plane table", p.N);
    l.block = dim3(kFwdTileW, kFwdTileH);
    l.grid = dim3((p.W + kFwdTileW - 1) / kFwdTileW, (p.H + kFwdTileH - 1) / kFwdTileH, p.V);
    if (l.grid.y > 65535) return fail(GMPI_ERR_UNSUPPORTED, "image height %d too large", p.H);
    if (p.V > 65535) return fail(GMPI_ERR_UNSUPPORTED, "V=%d views exceed one launch of the direct kernel (65535); split the batch", p.V);
    l.key = key;
    return GMPI_OK;
}

// Forward launch of a checked call (check_call).  occ: empty-space skipping against this occupancy map.
static int launch_fwd(RenderParams p, cudaStream_t st, const uint32_t* occ = nullptr) {
    if (p.V == 0) return GMPI_OK;
    // float4 epilogue stores: whole quads of x stay inside a row and every destination is 16-byte aligned.  Peer buffers are
    // symmetric-memory allocations (256-byte aligned bases; frame slabs are multiples of 16 bytes when W % 4 == 0).
    if (p.W % 4 == 0 && !p.video_rgb && (p.n_peers > 0 || (aligned16(p.color) && aligned16(p.depth)))) p.options |= kOptVec4Stores;
    Launch l(p);
    int rc = fwd_launch(l, occ);
    if (rc) return rc;
    // the direct kernel walks no stages: it loads per pixel, and composites every plane (which gives a skipping call's output)
    const unsigned long long walked = (unsigned long long)l.tiles * p.N;
    const KernelUnit& unit = key_unit(l.key);
    if ((p.options & GMPI_EARLY_STOP) && (rc = reset_stage_stats(kEarlyStopStats, unit, walked, st)) != 0) return rc;
    if (occ && (rc = reset_stage_stats(kSkipStats, unit, walked, st)) != 0) return rc;
    return launch(l, st);
}

static int zero_grads(const RenderParams& p, cudaStream_t st) {
    const size_t tex = (size_t)p.Ht * p.Wt;
    if (p.g_alpha) {
        GMPI_CUDA_OK(cudaMemsetAsync(p.g_rgb, 0, sizeof(float) * (size_t)p.M * 3 * tex, st));
        GMPI_CUDA_OK(cudaMemsetAsync(p.g_alpha, 0, sizeof(float) * (size_t)p.M * p.N * tex, st));
        if (p.g_bg_rgb) GMPI_CUDA_OK(cudaMemsetAsync(p.g_bg_rgb, 0, sizeof(float) * (size_t)p.M * 3 * tex, st));
    } else {
        GMPI_CUDA_OK(cudaMemsetAsync(p.g_rgba, 0, sizeof(float) * (size_t)p.M * p.N * 4 * tex, st));
    }
    return GMPI_OK;
}

// The GMPI_WHY_* bits of every reason the staged box backward is not launched for p (0 = box): the one decision behind launch_bwd,
// launch_bwd_deterministic (from the caller's descriptor) and gmpi_mpi_render_bwd_plan_ex.  The box kernel reads the MPI through the
// staged forward's tensor maps on its persistent grid, so every reason of fwd_why carries over; its own conditions are a saved
// transmittance, W % 4 == 0, 16-byte aligned gradient bases of the MPI's form and transmittance base (NULL counts as aligned), and
// V*N < 2^31 (pixel planes of the transmittance's tensor map).
static uint32_t bwd_why(const RenderParams& p) {
    uint32_t w = fwd_why(p);
    if (!p.transmittance) w |= GMPI_WHY_NO_TRANSMITTANCE;
    if (p.W % 4 != 0) w |= GMPI_WHY_IMG_WIDTH;
    const bool grads = factored(p) ? aligned16(p.g_rgb) && aligned16(p.g_alpha) && aligned16(p.g_bg_rgb) : aligned16(p.g_rgba);
    if (!grads || !aligned16(p.transmittance)) w |= GMPI_WHY_GRAD_ALIGNMENT;
    if ((size_t)p.V * p.N >= ((size_t)1 << 31)) w |= GMPI_WHY_MANY_PIXEL_PLANES;
    return w;
}

// The direct backward's CTA of a checked call: as many threads (<=128) as the per-thread transmittance stash allows, and its grid.
// Refuses what exceeds the kernel's limits; the launch and the plan query both take them from here.
static int bwd_direct_shape(const RenderParams& p, dim3& block, dim3& grid, size_t& smem) {
    int tile_w = 32, tile_h = 4;
    for (;; tile_h >>= 1) {
        if (tile_h == 0) return fail(GMPI_ERR_UNSUPPORTED, "N=%d planes exceed the backward stash (227 KB / 32 threads)", p.N);
        smem = sizeof(PlaneConst) * (size_t)p.N + sizeof(float) * (size_t)p.N * tile_w * tile_h;
        if (smem <= 227 * 1024) break;
    }
    block = dim3(tile_w, tile_h);
    grid = dim3((p.W + tile_w - 1) / tile_w, (p.H + tile_h - 1) / tile_h, p.V);
    if (grid.y > 65535) return fail(GMPI_ERR_UNSUPPORTED, "image height %d too large", p.H);
    if (p.V > 65535) return fail(GMPI_ERR_UNSUPPORTED, "V=%d views exceed one launch of the direct kernel (65535); split the batch", p.V);
    return GMPI_OK;
}

// The backward kernel of a checked call with V > 0, with its launch: the box kernel when `box` (bwd_why(p) == 0), else the two-pass
// direct kernel (any shape, no saved state).  det: the deterministic variant, adding into the sums of l.da.
static int bwd_launch(Launch& l, bool box, bool det) {
    const RenderParams& p = l.p;
    uint32_t key = kKeyBwd | (det ? kKeyDet : 0) | ((p.options & GMPI_ALIGN_CORNERS) ? kKeyAC : 0);
    if (box) {
        if (encode_mpi_maps(l.maps, p, kBwdMaxBH, BwdRing::kColourCopyRows) != 0) return fail(GMPI_ERR_CUDA, "cuTensorMapEncodeTiled failed");
        if (encode_slab_map(&l.maps.t, p.transmittance, ElemTraits<float>::kMap, (uint64_t)p.V * p.N, p.H, p.W, kTileW, kBwdTileH, 1) != 0)
            return fail(GMPI_ERR_CUDA, "cuTensorMapEncodeTiled (transmittance) failed");
        if (int rc = persistent_grid(l, kBwdTileH)) return rc;
        l.block = dim3(kBwdThreads);
        l.smem = kBwdSmem;
        key |= kKeyStaged | (factored(p) ? kKeyFac : 0);
    } else {
        if (int rc = bwd_direct_shape(p, l.block, l.grid, l.smem)) return rc;
        l.ints[0] = (int)l.block.x;
        l.ints[1] = (int)l.block.y;
        l.arg(&l.ints[0]);
        l.arg(&l.ints[1]);
    }
    if (det) l.arg(&l.da);
    l.key = key;
    return GMPI_OK;
}

static int launch_bwd(RenderParams p, cudaStream_t st) {
    const bool zero = (p.options & GMPI_ZERO_GRAD) != 0;
    if (p.V == 0) return zero ? zero_grads(p, st) : GMPI_OK;
    Launch l(p);
    int rc = bwd_launch(l, bwd_why(p) == 0, false);
    if (rc) return rc;
    if (zero && (rc = zero_grads(p, st)) != 0) return rc;
    return launch(l, st);
}

// ---- deterministic backward (DetAcc, DESIGN.md section 4.3) ----
// Scratch: a 256-byte header (the pre-pass's two bounds), the int64 sums of the G gradient elements (in the order g_rgba, or
// g_rgb | g_alpha | g_bg_rgb), then four non-finite bits per element.
struct DetLayout {
    size_t G, seg1, seg2, nf_off, bytes;     // seg1, seg2: first elements of g_alpha and g_bg_rgb (factored; G otherwise)
};
constexpr size_t kDetHeaderBytes = 256;
constexpr int kDetMinFixBits = 24;

// The layout of a call with checked sizes (check_call).
static int det_layout(const RenderParams& p, DetLayout& L) {
    const double tex = (double)p.Ht * p.Wt, M = p.M, N = p.N;
    const double G = factored(p) ? M * 3 * tex + M * N * tex + (p.bg_rgb ? M * 3 * tex : 0.0) : M * N * 4 * tex;
    if (G * 9 > 0x1p62) return fail(GMPI_ERR_UNSUPPORTED, "%.0f gradient elements exceed the deterministic scratch's range", G);
    const size_t t = (size_t)p.Ht * p.Wt;
    if (factored(p)) {
        L.seg1 = (size_t)p.M * 3 * t;
        L.seg2 = L.seg1 + (size_t)p.M * p.N * t;
        L.G = L.seg2 + (p.bg_rgb ? (size_t)p.M * 3 * t : 0);
    } else {
        L.G = L.seg1 = L.seg2 = (size_t)p.M * p.N * 4 * t;
    }
    L.nf_off = kDetHeaderBytes + 8 * L.G;
    L.bytes = L.nf_off + 4 * ((L.G + 7) / 8);
    return GMPI_OK;
}

static int ceil_log2(unsigned long long x) {
    int b = 0;
    while (b < 63 && (1ull << b) < x) ++b;
    return b;
}
// Fraction bits k of the unit 2^(E - k) for elements that sum `planes` planes: one (view, plane) adds at most H*W taps of bilinear
// weight <= 1 to an element, and V bounds the views of one MPI (view2mpi is device memory).  With C = H*W*V*planes taps of
// |c| <= 2^E w each, a sum is below 2^(k+1) C <= 2^62 in units of 2^(E - k) (DESIGN.md section 4.3): it cannot wrap int64.
static int det_fix_bits(const RenderParams& p, int planes) {
    return 61 - ceil_log2((unsigned long long)p.H * p.W) - ceil_log2((unsigned long long)p.V) - ceil_log2((unsigned long long)planes);
}

static int launch_bwd_deterministic(RenderParams p, void* scratch, size_t scratch_bytes, cudaStream_t st) {
    DetLayout L;
    int rc = det_layout(p, L);
    if (rc) return rc;
    if (!scratch) return fail(GMPI_ERR_INVALID_ARGUMENT, "null scratch pointer (gmpi_mpi_render_bwd_deterministic_scratch_bytes gives its size)");
    if (!aligned16(scratch)) return fail(GMPI_ERR_INVALID_ARGUMENT, "the scratch must be 16-byte aligned");
    if (scratch_bytes < L.bytes)
        return fail(GMPI_ERR_INVALID_ARGUMENT, "scratch of %zu bytes is smaller than the %zu bytes this call needs", scratch_bytes, L.bytes);
    const bool fac = factored(p);
    const int k_a = det_fix_bits(p, 1), k_rgb = det_fix_bits(p, fac ? p.N : 1);
    if (k_rgb < kDetMinFixBits)
        return fail(GMPI_ERR_UNSUPPORTED, "V=%d views of %dx%d pixels leave %d fraction bits for exact int64 sums (at least %d needed)", p.V,
                    p.H, p.W, k_rgb, kDetMinFixBits);
    if (p.V == 0) return (p.options & GMPI_ZERO_GRAD) ? zero_grads(p, st) : GMPI_OK;
    Launch l(p);
    DetAcc& da = l.da;
    char* s = static_cast<char*>(scratch);
    da.bounds = reinterpret_cast<uint32_t*>(s);
    da.acc = reinterpret_cast<unsigned long long*>(s + kDetHeaderBytes);
    da.base = reinterpret_cast<float*>(da.acc);
    da.nf = reinterpret_cast<uint32_t*>(s + L.nf_off);
    da.k_a = k_a;
    da.k_rgb = k_rgb;
    // the kernels' gradient pointers address the sums (DetAcc); the finish pass writes the caller's
    if (fac) {
        l.p.g_rgb = da.base;
        l.p.g_alpha = da.base + L.seg1;
        l.p.g_bg_rgb = p.g_bg_rgb ? da.base + L.seg2 : nullptr;
    } else {
        l.p.g_rgba = da.base;
    }
    if ((rc = bwd_launch(l, bwd_why(p) == 0, true)) != 0) return rc;
    GMPI_CUDA_OK(cudaMemsetAsync(scratch, 0, L.bytes, st));
    dim3 bgrid((unsigned)(((size_t)p.H * p.W + 255) / 256), (unsigned)(p.V < 65535 ? p.V : 65535));
    if ((rc = launch_kernel(mpi_bwd_det_bounds_kernel, bgrid, 256, 0, st, l.p, da.bounds)) != 0) return rc;
    if ((rc = launch(l, st)) != 0) return rc;
    int sms = 0;
    if ((rc = device_attr(cudaDevAttrMultiProcessorCount, &sms)) != 0) return rc;
    return launch_kernel(mpi_bwd_det_finish_kernel, sms * 8, 256, 0, st, da, fac ? p.g_rgb : p.g_rgba, p.g_alpha, p.g_bg_rgb, L.G, L.seg1,
                         L.seg2, (size_t)p.Ht * p.Wt, fac, (p.options & GMPI_ZERO_GRAD) != 0);
}

static RenderParams params_from_desc(const gmpi_render_desc* d) {
    RenderParams p{};
    p.rgba = d->rgba; p.rgb = d->rgb; p.alpha = d->alpha; p.bg_rgb = d->bg_rgb;
    p.view2mpi = d->view2mpi; p.dhw = d->dhw; p.ray_dir = d->ray_dir; p.eye = d->eye; p.z_dir = d->z_dir; p.cam = d->cam;
    p.color = d->color; p.depth = d->depth; p.transmittance = d->transmittance; p.flags = d->flags;
    p.peer_frames = d->peer_frames; p.n_peers = d->n_peers; p.frame_offset = d->frame_offset;
    p.video_rgb = d->video_rgb; p.video_depth = d->video_depth; p.depth_near = d->depth_near; p.depth_range = d->depth_range;
    p.g_color = d->g_color; p.g_depth = d->g_depth; p.g_rgba = d->g_rgba; p.g_rgb = d->g_rgb; p.g_bg_rgb = d->g_bg_rgb; p.g_alpha = d->g_alpha;
    p.M = d->M; p.V = d->V; p.N = d->N; p.Ht = d->Ht; p.Wt = d->Wt; p.H = d->H; p.W = d->W;
    p.view_group = d->view_group;
    p.options = d->options & 0xffffu;      // the upper bits are internal
    // a descriptor of the previous size (GMPI_RENDER_DESC_V2_BYTES) ends before early_stop: check_desc refused GMPI_EARLY_STOP there
    p.early_stop = d->struct_bytes == sizeof(gmpi_render_desc) ? d->early_stop : 0.0f;
    return p;
}

static int check_desc(const gmpi_render_desc* d) {
    if (!d) return fail(GMPI_ERR_INVALID_ARGUMENT, "null descriptor");
    if (d->struct_bytes != sizeof(gmpi_render_desc) && d->struct_bytes != GMPI_RENDER_DESC_V2_BYTES)
        return fail(GMPI_ERR_INVALID_ARGUMENT, "gmpi_render_desc.struct_bytes = %u, this library expects %zu or %zu (ABI %d)", d->struct_bytes,
                    sizeof(gmpi_render_desc), (size_t)GMPI_RENDER_DESC_V2_BYTES, GMPI_ABI_VERSION);
    if (d->struct_bytes != sizeof(gmpi_render_desc) && (d->options & GMPI_EARLY_STOP))
        return fail(GMPI_ERR_INVALID_ARGUMENT, "GMPI_EARLY_STOP needs struct_bytes = %zu (a descriptor with the early_stop field)",
                    sizeof(gmpi_render_desc));
    return GMPI_OK;
}

// The RenderParams p of a descriptor call, checked (check_desc, check_call).
static int check_desc_call(const gmpi_render_desc* d, const Call& c, RenderParams& p) {
    int rc = check_desc(d);
    if (rc) return rc;
    p = params_from_desc(d);
    return check_call(p, c);
}

// The path of gmpi_mpi_render_fwd_ex (kFwdCall) and gmpi_mpi_render_bwd_ex (kBwdCall).
static int render(const gmpi_render_desc* d, const Call& c) {
    RenderParams p{};
    int rc = check_desc_call(d, c, p);
    return rc ? rc : c.kind == kBwdCall ? launch_bwd(p, (cudaStream_t)d->stream) : launch_fwd(p, (cudaStream_t)d->stream);
}

// The descriptor of a classic entry point's arguments: an expanded fp32 MPI and the reference's ray tensors.  The entry point adds
// its outputs or gradients and takes the path of the descriptor call it corresponds to, checked as a classic call.
static gmpi_render_desc classic_desc(const float* rgba, const int32_t* view2mpi, const float* dhw, const float* ray_dir, const float* eye,
                                     const float* z_dir, int M, int V, int N, int Ht, int Wt, int H, int W, uint32_t options, void* stream) {
    gmpi_render_desc d{};
    d.struct_bytes = sizeof(gmpi_render_desc); d.options = options; d.view_group = 1; d.stream = stream;
    d.M = M; d.V = V; d.N = N; d.Ht = Ht; d.Wt = Wt; d.H = H; d.W = W;
    d.rgba = rgba; d.view2mpi = view2mpi; d.dhw = dhw; d.ray_dir = ray_dir; d.eye = eye; d.z_dir = z_dir;
    return d;
}

// The occupancy-map build of a checked call (mpi_kernel_keys.cuh), by element type and form.  The expanded fp32 and fp16 builds also
// set the range check's flags from the same loads; uint8 MPIs are expanded, and every code is inside [0, 1].  The kernels read the
// MPI as the bit patterns U of its elements.
template <class U> static const U* elem_bits(const float* mpi) { return reinterpret_cast<const U*>(mpi); }

static int occ_build(const RenderParams& p, uint32_t* map, int words, int rows, cudaStream_t st) {
    const int M = p.M, N = p.N, Ht = p.Ht, Wt = p.Wt;
    const dim3 block(32 * kOccB);
    if (factored(p)) {
        const dim3 grid(words, rows, M < 65535 ? M : 65535);
        if (p.options & GMPI_MPI_F16)
            return launch_kernel(gmpi_occ_factored_f16, grid, block, 0, st, elem_bits<uint16_t>(p.rgb), elem_bits<uint16_t>(p.bg_rgb),
                                 elem_bits<uint16_t>(p.alpha), map, M, N, Ht, Wt, words, rows);
        return launch_kernel(gmpi_occ_factored_f32, grid, block, 0, st, elem_bits<uint32_t>(p.rgb), elem_bits<uint32_t>(p.bg_rgb),
                             elem_bits<uint32_t>(p.alpha), map, M, N, Ht, Wt, words, rows);
    }
    const long long P = (long long)M * N;
    if (P > 0x7fffffffLL) return fail(GMPI_ERR_UNSUPPORTED, "%lld planes exceed the occupancy build (2^31)", P);
    const int planes = (int)P;
    const dim3 grid(words, rows, planes < 65535 ? planes : 65535);
    if (p.options & GMPI_MPI_U8)
        return launch_kernel(gmpi_occ_expanded_u8, grid, block, 0, st, elem_bits<uint8_t>(p.rgba), map, planes, Ht, Wt, words, rows);
    if (p.options & GMPI_MPI_F16)
        return launch_kernel(gmpi_occ_expanded_f16, grid, block, 0, st, elem_bits<uint16_t>(p.rgba), map, p.flags, planes, Ht, Wt, words, rows);
    return launch_kernel(gmpi_occ_expanded_f32, grid, block, 0, st, elem_bits<uint32_t>(p.rgba), map, p.flags, planes, Ht, Wt, words, rows);
}

// The range check of an fp32 or (f16) fp16 rgba: 16-byte loads when every slab is a whole number of them on an aligned base.
static int check_range(const void* rgba, bool f16, int M, int N, int Ht, int Wt, uint32_t* flags, cudaStream_t st) {
    if (!rgba || !flags) return fail(GMPI_ERR_INVALID_ARGUMENT, "null pointer");
    if (M < 1 || N < 1 || Ht < 1 || Wt < 1) return fail(GMPI_ERR_INVALID_ARGUMENT, "bad sizes");
    const size_t slab = (size_t)Ht * Wt, n_slabs = (size_t)M * N * 4;
    int sms = 132;
    if (int rc = device_attr(cudaDevAttrMultiProcessorCount, &sms)) return rc;
    const int grid = sms * 8;
    const auto run = [&](auto e) {
        using T = decltype(e);
        using E = typename T::Elem;
        using Bits = typename T::Bits;
        if (slab % T::kAlign == 0 && aligned16(rgba))
            return launch_kernel(mpi_check_range_kernel<E, uint4>, grid, 256, 0, st, static_cast<const uint4*>(rgba), n_slabs,
                                 slab / T::kAlign, flags);
        return launch_kernel(mpi_check_range_kernel<E, Bits>, grid, 256, 0, st, static_cast<const Bits*>(rgba), n_slabs, slab, flags);
    };
    return f16 ? run(ElemTraits<__half>{}) : run(ElemTraits<float>{});
}

extern "C" {

int gmpi_abi_version(void) { return GMPI_ABI_VERSION; }

const char* gmpi_last_error(void) { return g_err; }

int gmpi_debug_set_fwd_variant(int variant) {
    if (variant < 0 || variant > 2) return fail(GMPI_ERR_INVALID_ARGUMENT, "variant must be 0 (auto), 1 (direct) or 2 (staged)");
    g_fwd_variant.store(variant, std::memory_order_relaxed);
    return GMPI_OK;
}

int gmpi_debug_set_fwd_stages(int stages) {
    if (stages != 0 && stages != kStreamStages && stages != kStages)
        return fail(GMPI_ERR_INVALID_ARGUMENT, "stages must be 0 (auto), %d or %d", kStreamStages, kStages);
    g_fwd_stages.store(stages, std::memory_order_relaxed);
    return GMPI_OK;
}

int gmpi_debug_fwd_early_stop_stats(unsigned long long* skipped, unsigned long long* total) {
    return read_stage_stats(kEarlyStopStats, skipped, total);
}

int gmpi_debug_fwd_ring_stages(int M, int V, int N, int Ht, int Wt, int view_group) {
    if (M < 1 || V < 1 || N < 1 || Ht < 1 || Wt < 1 || view_group < 0)
        return -fail(GMPI_ERR_INVALID_ARGUMENT, "gmpi_debug_fwd_ring_stages: bad argument");
    RenderParams p{};
    p.M = M; p.V = V; p.N = N; p.Ht = Ht; p.Wt = Wt;
    p.view_group = view_group < 1 ? 1 : view_group;
    int l2 = 0, rc = device_attr(cudaDevAttrL2CacheSize, &l2);
    if (rc) return -rc;
    return fwd_ring_stages(p, l2);
}

// Host evaluation of the staged kernels' tile order (same TileWalk code): tiles of CTA `cta` in a grid of `grid` CTAs, as
// (view, px0, py0) triples.  Returns the count, or a negative error.
int gmpi_debug_tile_walk_ex(int H, int W, int V, int tile_h, int view_group, int grid, int cta, int* out_v_px0_py0, int max_tiles) {
    if (H < 1 || W < 1 || V < 1 || tile_h < 1 || grid < 1 || cta < 0 || cta >= grid || max_tiles < 0 || (max_tiles > 0 && !out_v_px0_py0))
        return -fail(GMPI_ERR_INVALID_ARGUMENT, "gmpi_debug_tile_walk: bad argument");
    TileWalk w;
    w.init((W + kTileW - 1) / kTileW, H, V, cta, grid, tile_h, view_group);
    TileXY t;
    int n = 0;
    for (; w.at(n, t); ++n)
        if (n < max_tiles) { out_v_px0_py0[3 * n] = t.v; out_v_px0_py0[3 * n + 1] = t.px0; out_v_px0_py0[3 * n + 2] = t.py0; }
    return n;
}

// Host evaluation of the expanded forward's copies of one stage (same code as the producer): for a footprint of n_rows staged rows
// (a multiple of 4, at most the ring's box height) writes (first row, rows) of every copy; returns their number.
int gmpi_debug_copy_plan(int n_rows, int* out_row_rows, int max_copies) {
    if (n_rows < 0 || n_rows % kRowsPerOp != 0 || n_rows > kMaxBH || max_copies < 0 || (max_copies > 0 && !out_row_rows))
        return -fail(GMPI_ERR_INVALID_ARGUMENT, "gmpi_debug_copy_plan: n_rows must be a multiple of %d in [0, %d]", kRowsPerOp, kMaxBH);
    int n = 0;
    for (int lane = 0; lane < 4; ++lane) {
        int before;
        const int h = binary_copy_of_lane(n_rows / kRowsPerOp, lane, before);
        if (!h) continue;
        if (n < max_copies) { out_row_rows[2 * n] = before * kRowsPerOp; out_row_rows[2 * n + 1] = h * kRowsPerOp; }
        ++n;
    }
    return n;
}

int gmpi_debug_tile_walk(int H, int W, int V, int grid, int cta, int* out_v_px0_py0, int max_tiles) {
    return gmpi_debug_tile_walk_ex(H, W, V, kTileH, 1, grid, cta, out_v_px0_py0, max_tiles);
}

int gmpi_mpi_render_fwd_plan(int V, int N, int Ht, int Wt, int H, int W, const void* rgba, uint32_t* why) {
    const gmpi_render_desc d = classic_desc(static_cast<const float*>(rgba), nullptr, nullptr, nullptr, nullptr, nullptr, 1, V, N, Ht, Wt,
                                            H, W, 0, nullptr);
    return gmpi_mpi_render_fwd_plan_ex(&d, why);
}

int gmpi_mpi_render_fwd_plan_ex(const gmpi_render_desc* d, uint32_t* why) {
    int rc = check_desc(d);
    if (rc) return -rc;
    const uint32_t w = fwd_why(params_from_desc(d));
    if (why) *why = w;
    return w == 0 ? GMPI_PLAN_STAGED : GMPI_PLAN_DIRECT;
}

int gmpi_mpi_render_bwd_plan_ex(const gmpi_render_desc* d, uint32_t* why) {
    RenderParams p{};
    int rc = check_desc_call(d, Call{kBwdPlanCall}, p);
    if (rc) return -rc;
    const uint32_t w = bwd_why(p);
    if (why) *why = w;
    // the direct kernel's limits refuse a call that launches it (launch_bwd: a call with V = 0 launches nothing)
    dim3 block, grid;
    size_t smem = 0;
    if (w != 0 && p.V > 0 && (rc = bwd_direct_shape(p, block, grid, smem)) != 0) return -rc;
    return w == 0 ? GMPI_PLAN_STAGED : GMPI_PLAN_DIRECT;
}

int gmpi_debug_last_render_key(int device, uint32_t* key) {
    if (!key) return fail(GMPI_ERR_INVALID_ARGUMENT, "null pointer");
    if (device < 0 || device >= kMaxKeyDevices) return fail(GMPI_ERR_INVALID_ARGUMENT, "device %d out of range", device);
    const uint64_t k = g_last_render_key[device].load(std::memory_order_relaxed);
    if (k == 0) return fail(GMPI_ERR_INVALID_ARGUMENT, "no render kernel was launched on device %d", device);
    *key = (uint32_t)(k - 1);
    return GMPI_OK;
}

const char* gmpi_mpi_render_fwd_variant(int N, int Ht, int Wt, int H, int W) {
    return gmpi_mpi_render_fwd_plan(1 << 20, N, Ht, Wt, H, W, nullptr, nullptr) == GMPI_PLAN_STAGED ? "fwd_staged_tma_64x30" : "fwd_direct_32x8";
}

int gmpi_mpi_render_fwd(const float* rgba, const int32_t* view2mpi, const float* dhw, const float* ray_dir,
                        const float* eye, const float* z_dir, float* color, float* depth, uint32_t* flags, int M,
                        int V, int N, int Ht, int Wt, int H, int W, uint32_t options, void* stream) {
    gmpi_render_desc d = classic_desc(rgba, view2mpi, dhw, ray_dir, eye, z_dir, M, V, N, Ht, Wt, H, W, options, stream);
    d.color = color; d.depth = depth; d.flags = flags;
    return render(&d, Call{kFwdCall, true});
}

int gmpi_mpi_render_fwd_train(const float* rgba, const int32_t* view2mpi, const float* dhw, const float* ray_dir,
                              const float* eye, const float* z_dir, float* color, float* depth, float* transmittance,
                              uint32_t* flags, int M, int V, int N, int Ht, int Wt, int H, int W, uint32_t options,
                              void* stream) {
    gmpi_render_desc d = classic_desc(rgba, view2mpi, dhw, ray_dir, eye, z_dir, M, V, N, Ht, Wt, H, W, options, stream);
    d.color = color; d.depth = depth; d.flags = flags; d.transmittance = transmittance;
    return render(&d, Call{kFwdCall, true, transmittance ? nullptr : "null transmittance buffer"});
}

int gmpi_mpi_render_fwd_gather(const float* rgba, const int32_t* view2mpi, const float* dhw, const float* ray_dir,
                               const float* eye, const float* z_dir, float* const* peer_frames, int n_peers,
                               int frame_offset, uint32_t* flags, int M, int V, int N, int Ht, int Wt, int H, int W,
                               uint32_t options, void* stream) {
    gmpi_render_desc d = classic_desc(rgba, view2mpi, dhw, ray_dir, eye, z_dir, M, V, N, Ht, Wt, H, W, options, stream);
    d.flags = flags; d.peer_frames = peer_frames; d.n_peers = n_peers; d.frame_offset = frame_offset;
    return render(&d, Call{kFwdCall, true, n_peers < 1 ? "n_peers must be >= 1" : nullptr});
}

int gmpi_mpi_render_bwd(const float* rgba, const int32_t* view2mpi, const float* dhw, const float* ray_dir,
                        const float* eye, const float* z_dir, const float* g_color, const float* g_depth,
                        float* g_rgba, int M, int V, int N, int Ht, int Wt, int H, int W, uint32_t options,
                        void* stream) {
    gmpi_render_desc d = classic_desc(rgba, view2mpi, dhw, ray_dir, eye, z_dir, M, V, N, Ht, Wt, H, W, options, stream);
    d.g_color = g_color; d.g_depth = g_depth; d.g_rgba = g_rgba;
    return render(&d, Call{kBwdCall, true});
}

int gmpi_mpi_render_bwd_saved(const float* rgba, const int32_t* view2mpi, const float* dhw, const float* ray_dir,
                              const float* eye, const float* z_dir, const float* transmittance, const float* g_color,
                              const float* g_depth, float* g_rgba, int M, int V, int N, int Ht, int Wt, int H, int W,
                              uint32_t options, void* stream) {
    gmpi_render_desc d = classic_desc(rgba, view2mpi, dhw, ray_dir, eye, z_dir, M, V, N, Ht, Wt, H, W, options, stream);
    d.g_color = g_color; d.g_depth = g_depth; d.g_rgba = g_rgba; d.transmittance = const_cast<float*>(transmittance);
    return render(&d, Call{kBwdCall, true, transmittance ? nullptr : "null gradient / transmittance pointer"});
}

int gmpi_mpi_zero_async(void* ptr, size_t bytes, void* stream) {
    if (!ptr && bytes) return fail(GMPI_ERR_INVALID_ARGUMENT, "null pointer");
    GMPI_CUDA_OK(cudaMemsetAsync(ptr, 0, bytes, (cudaStream_t)stream));
    return GMPI_OK;
}

int gmpi_mpi_render_fwd_ex(const gmpi_render_desc* d) { return render(d, Call{kFwdCall}); }

int gmpi_mpi_render_bwd_ex(const gmpi_render_desc* d) { return render(d, Call{kBwdCall}); }

long long gmpi_mpi_render_bwd_deterministic_scratch_bytes(const gmpi_render_desc* d) {
    RenderParams p{};
    DetLayout L;
    int rc = check_desc_call(d, Call{kScratchCall}, p);
    if (rc || (rc = det_layout(p, L)) != 0) return -rc;
    return (long long)L.bytes;
}

int gmpi_mpi_render_bwd_deterministic_ex(const gmpi_render_desc* d, void* scratch, size_t scratch_bytes) {
    RenderParams p{};
    int rc = check_desc_call(d, Call{kBwdCall}, p);
    return rc ? rc : launch_bwd_deterministic(p, scratch, scratch_bytes, (cudaStream_t)d->stream);
}

long long gmpi_mpi_occupancy_bytes(const gmpi_render_desc* d) {
    RenderParams p{};
    int rc = check_desc_call(d, Call{kOccQueryCall}, p);
    return rc ? -rc : (long long)occ_map_bytes(p);
}

int gmpi_mpi_build_occupancy(const gmpi_render_desc* d, void* occ, size_t bytes) {
    RenderParams p{};
    int rc = check_desc_call(d, Call{kOccBuildCall, false, nullptr, occ, bytes}, p);
    if (rc) return rc;
    const int words = occ_words(p.Wt), rows = occ_rows(p.Ht);
    if (rows > 65535) return fail(GMPI_ERR_UNSUPPORTED, "Ht=%d exceeds the occupancy build's grid (%d texel rows)", p.Ht, 65535 * kOccB);
    return occ_build(p, static_cast<uint32_t*>(occ), words, rows, (cudaStream_t)d->stream);
}

int gmpi_mpi_render_fwd_skip_ex(const gmpi_render_desc* d, const void* occ, size_t bytes) {
    RenderParams p{};
    int rc = check_desc_call(d, Call{kSkipCall, false, nullptr, occ, bytes}, p);
    return rc ? rc : launch_fwd(p, (cudaStream_t)d->stream, static_cast<const uint32_t*>(occ));
}

int gmpi_debug_fwd_skip_stats(unsigned long long* skipped, unsigned long long* total) {
    return read_stage_stats(kSkipStats, skipped, total);
}

// Host evaluation of the producer's box-versus-map test (same code, occ_box_bits, over the 32 lanes of the warp).
int gmpi_debug_box_occupied(const uint32_t* plane_map, int Ht, int Wt, int bx0, int by0, int bw, int rows) {
    if (!plane_map || Ht < 1 || Wt < 1 || bw < 1 || rows < 1)
        return -fail(GMPI_ERR_INVALID_ARGUMENT, "gmpi_debug_box_occupied: bad argument");
    uint32_t any = 0;
    for (int lane = 0; lane < 32; ++lane) any |= occ_box_bits(plane_map, Ht, Wt, occ_words(Wt), bx0, by0, bw, rows, lane);
    return any != 0;
}

int gmpi_debug_u8_codes_host(float* out) {
    if (!out) return fail(GMPI_ERR_INVALID_ARGUMENT, "null pointer");
    for (int b = 0; b < 256; ++b) out[b] = to_f32((uint8_t)b);
    return GMPI_OK;
}

int gmpi_debug_u8_codes(float* out, void* stream) {
    if (!out) return fail(GMPI_ERR_INVALID_ARGUMENT, "null pointer");
    return launch_kernel(gmpi_u8_codes, 1, 256, 0, (cudaStream_t)stream, out);
}

int gmpi_mpi_check_range(const float* rgba, int M, int N, int Ht, int Wt, uint32_t* flags, void* stream) {
    return check_range(rgba, false, M, N, Ht, Wt, flags, (cudaStream_t)stream);
}

int gmpi_mpi_check_range_f16(const void* rgba, int M, int N, int Ht, int Wt, uint32_t* flags, void* stream) {
    return check_range(rgba, true, M, N, Ht, Wt, flags, (cudaStream_t)stream);
}

int gmpi_debug_plane_coords(const int32_t* view2mpi, const float* dhw, const float* ray_dir, const float* eye,
                            float* out, int V, int N, int Ht, int Wt, int H, int W, uint32_t options, void* stream) {
    if (!view2mpi || !dhw || !ray_dir || !eye || !out) return fail(GMPI_ERR_INVALID_ARGUMENT, "null pointer");
    if (V < 1 || N < 1 || Ht < 1 || Wt < 1 || H < 1 || W < 1) return fail(GMPI_ERR_INVALID_ARGUMENT, "bad sizes");
    cudaStream_t st = (cudaStream_t)stream;
    const size_t img = (size_t)H * W;
    dim3 grid((unsigned)((img + 255) / 256), V);
    const auto kernel = (options & GMPI_ALIGN_CORNERS) ? mpi_debug_coords_kernel<true> : mpi_debug_coords_kernel<false>;
    return launch_kernel(kernel, grid, 256, 0, st, view2mpi, dhw, ray_dir, eye, out, V, N, Ht, Wt, H, W);
}

int gmpi_debug_plane_coords_packed(const int32_t* view2mpi, const float* dhw, const float* ray_dir, const float* eye,
                                   float* out, int V, int N, int Ht, int Wt, int H, int W, uint32_t options, void* stream) {
    if (!view2mpi || !dhw || !ray_dir || !eye || !out) return fail(GMPI_ERR_INVALID_ARGUMENT, "null pointer");
    if (V < 1 || N < 1 || Ht < 1 || Wt < 1 || H < 1 || W < 1 || ((size_t)H * W) % 2) return fail(GMPI_ERR_INVALID_ARGUMENT, "bad sizes");
    cudaStream_t st = (cudaStream_t)stream;
    const size_t pairs = (size_t)H * W / 2;
    dim3 grid((unsigned)((pairs + 255) / 256), V);
    const auto kernel = (options & GMPI_ALIGN_CORNERS) ? mpi_debug_coords_packed_kernel<true> : mpi_debug_coords_packed_kernel<false>;
    return launch_kernel(kernel, grid, 256, 0, st, view2mpi, dhw, ray_dir, eye, out, V, N, Ht, Wt, H, W);
}

int gmpi_debug_division(const float* a, const float* b, float* out_fast, float* out_ieee, size_t n, void* stream) {
    if (!a || !b || !out_fast || !out_ieee) return fail(GMPI_ERR_INVALID_ARGUMENT, "null pointer");
    return launch_kernel(mpi_debug_division_kernel, 1184, 256, 0, (cudaStream_t)stream, a, b, out_fast, out_ieee, n);
}

int gmpi_debug_cam_rays(const float* cam, float* ray_dir, int V, int H, int W, void* stream) {
    if (!cam || !ray_dir || V < 1 || H < 1 || W < 1) return fail(GMPI_ERR_INVALID_ARGUMENT, "bad argument");
    dim3 grid((unsigned)(((size_t)H * W + 255) / 256), V);
    return launch_kernel(mpi_debug_cam_rays_kernel, grid, 256, 0, (cudaStream_t)stream, cam, ray_dir, V, H, W);
}

// ------------------------------------------------------------------------------------------
// LightRenderer kernels (gmpi/core/light_renderer.py), SURVEY.md 8(f) N3
// ------------------------------------------------------------------------------------------
static int check_alpha_view(const float* alpha, long long mpi_stride, long long plane_stride, int M, int N, int Ht, int Wt) {
    if (!alpha) return fail(GMPI_ERR_INVALID_ARGUMENT, "null pointer");
    if (M < 1 || N < 1 || Ht < 1 || Wt < 1 || M > 65535) return fail(GMPI_ERR_INVALID_ARGUMENT, "bad sizes");
    if (((size_t)Ht * Wt) % 4 != 0 || plane_stride % 4 != 0 || mpi_stride % 4 != 0 || ((uintptr_t)alpha & 15) != 0)
        return fail(GMPI_ERR_UNSUPPORTED, "alpha planes must be 16-byte aligned with Ht*Wt %% 4 == 0 (float4 streaming)");
    return GMPI_OK;
}

int gmpi_mpi_alpha_depth_fwd(const float* alpha, long long mpi_stride, long long plane_stride, const float* plane_d, float* depth,
                             float* transmittance, int M, int N, int Ht, int Wt, void* stream) {
    int rc = check_alpha_view(alpha, mpi_stride, plane_stride, M, N, Ht, Wt);
    if (rc) return rc;
    if (!plane_d || !depth) return fail(GMPI_ERR_INVALID_ARGUMENT, "null pointer");
    const long long tex4 = (long long)Ht * Wt / 4;
    AlphaView a{alpha, mpi_stride, plane_stride};
    dim3 grid((unsigned)((tex4 + 255) / 256), M);
    const auto kernel = transmittance ? mpi_alpha_depth_fwd_kernel<true> : mpi_alpha_depth_fwd_kernel<false>;
    return launch_kernel(kernel, grid, 256, 0, (cudaStream_t)stream, a, plane_d, depth, transmittance, N, tex4);
}

int gmpi_mpi_alpha_depth_bwd(const float* alpha, long long mpi_stride, long long plane_stride, const float* plane_d,
                             const float* transmittance, const float* g_depth, float* g_alpha, long long g_mpi_stride,
                             long long g_plane_stride, int M, int N, int Ht, int Wt, void* stream) {
    int rc = check_alpha_view(alpha, mpi_stride, plane_stride, M, N, Ht, Wt);
    if (rc) return rc;
    if (!plane_d || !transmittance || !g_depth || !g_alpha) return fail(GMPI_ERR_INVALID_ARGUMENT, "null pointer");
    if (g_plane_stride % 4 != 0 || g_mpi_stride % 4 != 0 || ((uintptr_t)g_alpha & 15) != 0)
        return fail(GMPI_ERR_UNSUPPORTED, "g_alpha planes must be 16-byte aligned");
    const long long tex4 = (long long)Ht * Wt / 4;
    AlphaView a{alpha, mpi_stride, plane_stride};
    dim3 grid((unsigned)((tex4 + 255) / 256), M);
    return launch_kernel(mpi_alpha_depth_bwd_kernel, grid, 256, 0, (cudaStream_t)stream, a, plane_d, transmittance, g_depth, g_alpha,
                         g_mpi_stride, g_plane_stride, N, tex4);
}

int gmpi_mpi_apply_shading_fwd(const float* rgba, const float* shade, float* out, int M, int N, int Ht, int Wt, void* stream) {
    if (!rgba || !shade || !out) return fail(GMPI_ERR_INVALID_ARGUMENT, "null pointer");
    if (M < 1 || N < 1 || Ht < 1 || Wt < 1 || M > 65535 || N > 65535) return fail(GMPI_ERR_INVALID_ARGUMENT, "bad sizes");
    if (((size_t)Ht * Wt) % 4 != 0 || (((uintptr_t)rgba | (uintptr_t)shade | (uintptr_t)out) & 15) != 0)
        return fail(GMPI_ERR_UNSUPPORTED, "tensors must be 16-byte aligned with Ht*Wt %% 4 == 0 (float4 streaming)");
    const long long tex4 = (long long)Ht * Wt / 4;
    dim3 grid((unsigned)((tex4 + 255) / 256), N, M);
    return launch_kernel(mpi_apply_shading_fwd_kernel, grid, 256, 0, (cudaStream_t)stream, rgba, shade, out, N, tex4);
}

int gmpi_mpi_apply_shading_bwd(const float* rgba, const float* shade, const float* g_out, float* g_rgba, float* g_shade, int M, int N,
                               int Ht, int Wt, void* stream) {
    if (!rgba || !shade || !g_out || !g_rgba || !g_shade) return fail(GMPI_ERR_INVALID_ARGUMENT, "null pointer");
    if (M < 1 || N < 1 || Ht < 1 || Wt < 1 || M > 65535) return fail(GMPI_ERR_INVALID_ARGUMENT, "bad sizes");
    if (((size_t)Ht * Wt) % 4 != 0 ||
        (((uintptr_t)rgba | (uintptr_t)shade | (uintptr_t)g_out | (uintptr_t)g_rgba | (uintptr_t)g_shade) & 15) != 0)
        return fail(GMPI_ERR_UNSUPPORTED, "tensors must be 16-byte aligned with Ht*Wt %% 4 == 0 (float4 streaming)");
    const long long tex4 = (long long)Ht * Wt / 4;
    dim3 grid((unsigned)((tex4 + 255) / 256), M);
    return launch_kernel(mpi_apply_shading_bwd_kernel, grid, 256, 0, (cudaStream_t)stream, rgba, shade, g_out, g_rgba, g_shade, N, tex4);
}

// ------------------------------------------------------------------------------------------
// host-buffer entry points
// ------------------------------------------------------------------------------------------
// Per-device staging cache (grow-only; released by gmpi_mpi_release_host_cache or at exit): two MPI slots (the copy of MPI m+1
// overlaps the render of MPI m), per-view inputs/outputs, two streams, four events.
struct HostCache {
    float* mpi[2] = {nullptr, nullptr};
    size_t mpi_bytes = 0;
    void* misc = nullptr;           // dhw | ray/cam | eye | z | color | depth | video | v2m | flags, carved from one allocation
    size_t misc_bytes = 0;
    cudaStream_t s_copy = nullptr, s_run = nullptr;
    cudaEvent_t ev_in[2] = {nullptr, nullptr}, ev_free[2] = {nullptr, nullptr};
};
static HostCache g_host_cache[64];
static std::mutex g_host_mutex[64];     // one call at a time per device: the staging buffers are shared state

static void host_cache_release(HostCache& c) {
    for (int k = 0; k < 2; ++k) {
        if (c.mpi[k]) cudaFree(c.mpi[k]);
        if (c.ev_in[k]) cudaEventDestroy(c.ev_in[k]);
        if (c.ev_free[k]) cudaEventDestroy(c.ev_free[k]);
    }
    if (c.misc) cudaFree(c.misc);
    if (c.s_copy) cudaStreamDestroy(c.s_copy);
    if (c.s_run) cudaStreamDestroy(c.s_run);
    c = HostCache();
}

int gmpi_mpi_release_host_cache(void) {
    int cur = 0;
    cudaGetDevice(&cur);
    for (int d = 0; d < 64; ++d) {
        std::lock_guard<std::mutex> lock(g_host_mutex[d]);
        HostCache& c = g_host_cache[d];
        if (!c.misc && !c.mpi[0] && !c.s_run) continue;
        cudaSetDevice(d);
        host_cache_release(c);
    }
    cudaSetDevice(cur);
    return GMPI_OK;
}

// `h` holds HOST pointers (a checked call).  Streams every MPI through a double-buffered device slot and renders its views.
static int host_render_locked(HostCache& c, const RenderParams& h) {
    int rc = GMPI_OK;
    const int M = h.M, V = h.V, N = h.N, H = h.H, W = h.W;
    const size_t tex = (size_t)h.Ht * h.Wt, img = (size_t)H * W;
    const bool fac = factored(h), video = h.video_rgb != nullptr;
    // one slot = one MPI: expanded [N,4,tex], or factored rgb [3,tex] | bg [3,tex] | alpha [N,tex]
    // (offsets in MPI elements, of ebytes bytes each)
    const size_t ebytes = with_mpi_elem(h.options, [](auto e) { return sizeof(typename decltype(e)::Elem); });
    const size_t o_bg = 3 * tex, o_alpha = h.bg_rgb ? 6 * tex : 3 * tex;
    const size_t mpi_bytes = ebytes * (fac ? o_alpha + (size_t)N * tex : (size_t)N * 4 * tex);
    auto up = [](size_t x) { return (x + 255) & ~(size_t)255; };
    const size_t o_dhw = 0, o_ray = o_dhw + up(sizeof(float) * (size_t)M * N * 3),
                 o_eye = o_ray + up(h.cam ? sizeof(float) * (size_t)V * 16 : sizeof(float) * (size_t)V * 3 * img),
                 o_z = o_eye + up(sizeof(float) * (size_t)V * 3), o_color = o_z + up(sizeof(float) * (size_t)V * 3),
                 o_depth = o_color + up(video ? (size_t)V * 3 * img : sizeof(float) * (size_t)V * 3 * img),
                 o_v2m = o_depth + up(video ? (size_t)V * img : sizeof(float) * (size_t)V * img),
                 o_flags = o_v2m + up(sizeof(int32_t) * (size_t)(V > 0 ? V : 1)), misc_bytes = o_flags + 256;
    if (!c.s_run) {
        GMPI_CUDA_OK(cudaStreamCreateWithFlags(&c.s_copy, cudaStreamNonBlocking));
        GMPI_CUDA_OK(cudaStreamCreateWithFlags(&c.s_run, cudaStreamNonBlocking));
        for (int k = 0; k < 2; ++k) {
            GMPI_CUDA_OK(cudaEventCreateWithFlags(&c.ev_in[k], cudaEventDisableTiming));
            GMPI_CUDA_OK(cudaEventCreateWithFlags(&c.ev_free[k], cudaEventDisableTiming));
        }
    }
    if (c.mpi_bytes < mpi_bytes) {
        for (int k = 0; k < 2; ++k) {
            if (c.mpi[k]) GMPI_CUDA_OK(cudaFree(c.mpi[k]));
            c.mpi[k] = nullptr;
        }
        c.mpi_bytes = 0;
        for (int k = 0; k < 2; ++k) GMPI_CUDA_OK(cudaMalloc(&c.mpi[k], mpi_bytes));
        c.mpi_bytes = mpi_bytes;
    }
    if (c.misc_bytes < misc_bytes) {
        if (c.misc) GMPI_CUDA_OK(cudaFree(c.misc));
        c.misc = nullptr; c.misc_bytes = 0;
        GMPI_CUDA_OK(cudaMalloc(&c.misc, misc_bytes));
        c.misc_bytes = misc_bytes;
    }
    char* base = static_cast<char*>(c.misc);
    float *d_dhw = (float*)(base + o_dhw), *d_ray = (float*)(base + o_ray), *d_eye = (float*)(base + o_eye), *d_z = (float*)(base + o_z);
    int32_t* d_v2m = (int32_t*)(base + o_v2m);
    uint32_t* d_flags = (uint32_t*)(base + o_flags);
    cudaStream_t s_copy = c.s_copy, s_run = c.s_run;
    GMPI_CUDA_OK(cudaMemsetAsync(d_flags, 0, sizeof(uint32_t), s_run));
    GMPI_CUDA_OK(cudaMemsetAsync(d_v2m, 0, sizeof(int32_t) * (size_t)(V > 0 ? V : 1), s_run));   // a staged MPI is slot-local index 0
    GMPI_CUDA_OK(cudaMemcpyAsync(d_dhw, h.dhw, sizeof(float) * (size_t)M * N * 3, cudaMemcpyHostToDevice, s_run));
    if (h.cam) {
        GMPI_CUDA_OK(cudaMemcpyAsync(d_ray, h.cam, sizeof(float) * (size_t)V * 16, cudaMemcpyHostToDevice, s_run));
    } else {
        GMPI_CUDA_OK(cudaMemcpyAsync(d_ray, h.ray_dir, sizeof(float) * (size_t)V * 3 * img, cudaMemcpyHostToDevice, s_run));
        GMPI_CUDA_OK(cudaMemcpyAsync(d_eye, h.eye, sizeof(float) * (size_t)V * 3, cudaMemcpyHostToDevice, s_run));
        GMPI_CUDA_OK(cudaMemcpyAsync(d_z, h.z_dir, sizeof(float) * (size_t)V * 3, cudaMemcpyHostToDevice, s_run));
    }
    int v0 = 0, slot = 0, used[2] = {0, 0};
    for (int m = 0; m < M; ++m) {
        int v1 = v0;
        while (v1 < V && h.view2mpi[v1] == m) ++v1;
        if (v1 == v0) continue;
        if (used[slot]) GMPI_CUDA_OK(cudaStreamWaitEvent(s_copy, c.ev_free[slot], 0));
        char* d_mpi = reinterpret_cast<char*>(c.mpi[slot]);
        auto src = [ebytes](const float* base, size_t elems) { return reinterpret_cast<const char*>(base) + ebytes * elems; };
        if (fac) {
            GMPI_CUDA_OK(cudaMemcpyAsync(d_mpi, src(h.rgb, (size_t)m * 3 * tex), ebytes * 3 * tex, cudaMemcpyHostToDevice, s_copy));
            if (h.bg_rgb)
                GMPI_CUDA_OK(cudaMemcpyAsync(d_mpi + ebytes * o_bg, src(h.bg_rgb, (size_t)m * 3 * tex), ebytes * 3 * tex, cudaMemcpyHostToDevice, s_copy));
            GMPI_CUDA_OK(cudaMemcpyAsync(d_mpi + ebytes * o_alpha, src(h.alpha, (size_t)m * N * tex), ebytes * (size_t)N * tex, cudaMemcpyHostToDevice, s_copy));
        } else {
            GMPI_CUDA_OK(cudaMemcpyAsync(d_mpi, src(h.rgba, (size_t)m * N * 4 * tex), mpi_bytes, cudaMemcpyHostToDevice, s_copy));
        }
        GMPI_CUDA_OK(cudaEventRecord(c.ev_in[slot], s_copy));
        GMPI_CUDA_OK(cudaStreamWaitEvent(s_run, c.ev_in[slot], 0));
        RenderParams p = h;
        p.M = 1; p.V = v1 - v0;
        const auto at = [d_mpi, ebytes](size_t elems) { return reinterpret_cast<const float*>(d_mpi + ebytes * elems); };
        if (fac) { p.rgb = at(0); p.bg_rgb = h.bg_rgb ? at(o_bg) : nullptr; p.alpha = at(o_alpha); p.rgba = nullptr; }
        else p.rgba = at(0);
        p.view2mpi = d_v2m; p.dhw = d_dhw + (size_t)m * N * 3;
        // mpi.py:70 compares every plane distance with the eye of the CALL's view 0, not of this launch's first view
        if (h.cam) { p.cam = d_ray + (size_t)v0 * 16; p.eye0 = d_ray + 13; p.ray_dir = p.eye = p.z_dir = nullptr; }
        else { p.ray_dir = d_ray + (size_t)v0 * 3 * img; p.eye = d_eye + (size_t)v0 * 3; p.z_dir = d_z + (size_t)v0 * 3; p.eye0 = d_eye; }
        if (video) {
            p.video_rgb = (uint8_t*)(base + o_color) + (size_t)v0 * 3 * img;
            p.video_depth = h.video_depth ? (uint8_t*)(base + o_depth) + (size_t)v0 * img : nullptr;
            p.color = p.depth = nullptr;
        } else {
            p.color = (float*)(base + o_color) + (size_t)v0 * 3 * img;
            p.depth = (float*)(base + o_depth) + (size_t)v0 * img;
        }
        p.flags = d_flags;
        p.view_group = (M == 1 && h.view_group > 1) ? h.view_group : 1;
        rc = launch_fwd(p, s_run);
        if (rc) return rc;
        GMPI_CUDA_OK(cudaEventRecord(c.ev_free[slot], s_run));
        used[slot] = 1;
        slot ^= 1;
        v0 = v1;
    }
    if (video) {
        GMPI_CUDA_OK(cudaMemcpyAsync(h.video_rgb, base + o_color, (size_t)V * 3 * img, cudaMemcpyDeviceToHost, s_run));
        if (h.video_depth) GMPI_CUDA_OK(cudaMemcpyAsync(h.video_depth, base + o_depth, (size_t)V * img, cudaMemcpyDeviceToHost, s_run));
    } else {
        GMPI_CUDA_OK(cudaMemcpyAsync(h.color, base + o_color, sizeof(float) * (size_t)V * 3 * img, cudaMemcpyDeviceToHost, s_run));
        GMPI_CUDA_OK(cudaMemcpyAsync(h.depth, base + o_depth, sizeof(float) * (size_t)V * img, cudaMemcpyDeviceToHost, s_run));
    }
    GMPI_CUDA_OK(cudaMemcpyAsync(h.flags, d_flags, sizeof(uint32_t), cudaMemcpyDeviceToHost, s_run));
    GMPI_CUDA_OK(cudaStreamSynchronize(s_run));
    GMPI_CUDA_OK(cudaStreamSynchronize(s_copy));
    return GMPI_OK;
}

// The path of gmpi_mpi_render_host_ex: d's pointers are host memory, d->flags receives the flag word.
static int render_host(const gmpi_render_desc* d, int device, const Call& call) {
    RenderParams h{};
    int rc = check_desc_call(d, call, h);
    if (rc) return rc;
    if (device < 0 || device >= 64) return fail(GMPI_ERR_INVALID_ARGUMENT, "device %d out of range", device);
    for (int v = 0; v + 1 < h.V; ++v)
        if (h.view2mpi[v] > h.view2mpi[v + 1]) return fail(GMPI_ERR_INVALID_ARGUMENT, "views must be MPI-major (sorted view2mpi)");
    for (int v = 0; v < h.V; ++v)
        if (h.view2mpi[v] < 0 || h.view2mpi[v] >= h.M) return fail(GMPI_ERR_INVALID_ARGUMENT, "view2mpi[%d]=%d out of range", v, h.view2mpi[v]);
    GMPI_CUDA_OK(cudaSetDevice(device));
    std::lock_guard<std::mutex> lock(g_host_mutex[device]);
    HostCache& c = g_host_cache[device];
    rc = host_render_locked(c, h);
    if (rc != GMPI_OK) {
        // An error may have left asynchronous copies reading the caller's host buffers or rendering from the staging slots:
        // drain both streams before returning so that the caller may free its buffers and the next call starts clean.
        char keep[sizeof(g_err)];
        memcpy(keep, g_err, sizeof(keep));
        if (c.s_run) cudaStreamSynchronize(c.s_run);
        if (c.s_copy) cudaStreamSynchronize(c.s_copy);
        cudaGetLastError();
        memcpy(g_err, keep, sizeof(keep));
    }
    return rc;
}

int gmpi_mpi_render_fwd_host(const float* rgba, const int32_t* view2mpi, const float* dhw, const float* ray_dir,
                             const float* eye, const float* z_dir, float* color, float* depth, uint32_t* flags_out,
                             int M, int V, int N, int Ht, int Wt, int H, int W, uint32_t options, int device) {
    gmpi_render_desc d = classic_desc(rgba, view2mpi, dhw, ray_dir, eye, z_dir, M, V, N, Ht, Wt, H, W, options, nullptr);
    d.color = color; d.depth = depth; d.flags = flags_out;
    return render_host(&d, device, Call{kHostCall, true});
}

int gmpi_mpi_render_host_ex(const gmpi_render_desc* d, int device) { return render_host(d, device, Call{kHostCall}); }

}  // extern "C"
