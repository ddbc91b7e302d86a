/*
 * gmpi_mpi_render.h -- C ABI of the H100 (sm_90a) multiplane-image renderer.
 *
 * Drop-in boundary for ONE path of apple/ml-gmpi: the over-composite render of
 * gmpi/core/mpi.py (MPI.forward :308-436 + homography :26-153) as driven by
 * MPIRenderer.render (gmpi/core/mpi_renderer.py:387-469).  The reference has no FFI for this
 * path (it is a chain of ~30 ATen kernels); these entry points are what a binding for it binds.
 * INTEGRATION.md shows the ctypes stub and the two-line patch on the reference side.
 *
 * Conventions
 *   - plain C, plain pointers and sizes; no torch types.  All tensors fp32, contiguous,
 *     row-major, on the CUDA device that is current on the calling thread (except *_host).
 *   - `stream` is a cudaStream_t passed as void* (NULL = the legacy default stream).  All device
 *     entry points are asynchronous on that stream and allocate nothing.
 *   - return value: GMPI_OK, or an error code with a message available from gmpi_last_error()
 *     (thread-local).  The library never exits the process (the reference calls sys.exit(1) when
 *     rays leave the last plane, mpi.py:122-128; here that is a flag bit).
 *
 * Layouts (names follow the reference)
 *   rgba      [M, N, 4, Ht, Wt]  MPI textures in [0,1], planes ordered near -> far (mpi.py:413)
 *   dhw       [M, N, 3]          per plane: distance, metric height, metric width (mpi.py:59-63)
 *   view2mpi  [V] int32          MPI index of every rendered view.  Replaces the expand+cat of
 *                                mpi.py:334-346 (no copy of the MPI per view); views are
 *                                MPI-major like the reference's concatenation.
 *   ray_dir   [V, 3, H, W]       world-space unit rays per pixel (camera.py:182-211)
 *   eye       [V, 3]             camera position (camera.py:189)
 *   z_dir     [V, 3]             optical axis (camera.py:209)
 *   color     [V, 3, H, W]       composited colour in [0,1] (or 2c-1 if GMPI_COLOR_MINUS1_1)
 *   depth     [V, 1, H, W]       transmittance-weighted z-depth (mpi.py:434)
 *   flags     [1] uint32         OR-ed GMPI_FLAG_* bits (device memory; caller zeroes it)
 */
#ifndef GMPI_MPI_RENDER_H_
#define GMPI_MPI_RENDER_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define GMPI_ABI_VERSION 2

/* return codes */
#define GMPI_OK 0
#define GMPI_ERR_INVALID_ARGUMENT 1
#define GMPI_ERR_CUDA 2
#define GMPI_ERR_UNSUPPORTED 3

/* flag bits written to *flags: the reference's data-dependent asserts, reported instead of raised */
#define GMPI_FLAG_RGBA_RANGE 1u        /* rgba outside [0,1]            mpi_renderer.py:447-449 */
#define GMPI_FLAG_ALPHA_RANGE 2u       /* alpha outside [0,1]           mpi.py:185-187          */
#define GMPI_FLAG_LAST_PLANE_OOB 4u    /* |u| or |v| > 1 on last plane  mpi.py:103-109,381-395  */
#define GMPI_FLAG_PLANE_BEHIND_EYE 8u  /* !(distance >= z_eye[0])       mpi.py:70-72            */
                                       /*   over the planes of the MPIs some view renders; z_eye[0]: view 0's eye */

/* option bits for `options` */
#define GMPI_ALIGN_CORNERS 1u          /* MPI(align_corners=True), configs/gmpi.yml:74          */
#define GMPI_CHECK_LAST_PLANE 2u       /* assert_not_out_of_last_plane, mpi.py:317              */
#define GMPI_COLOR_MINUS1_1 4u         /* fuse "2*color-1" of mpi_renderer.py:467 into the store */
#define GMPI_ZERO_GRAD 8u              /* bwd: zero the gradient buffers on the stream before accumulating */
#define GMPI_U8_ROUND_HALF_UP 16u       /* uint8 epilogue: clamp, x*255+0.5 (torchvision save_image, fid_evaluation.py:125-130)
                                          instead of numpy's truncating astype (render_video.py:119-126) */
#define GMPI_EARLY_STOP 32u            /* forward only: early ray termination at gmpi_render_desc.early_stop (see there) */
#define GMPI_MPI_F16 64u               /* forward only: the descriptor's MPI tensors are IEEE binary16 (see gmpi_render_desc) */
#define GMPI_MPI_U8 128u               /* forward only: the descriptor's rgba is uint8, code b = b / 255 (see gmpi_render_desc) */

int gmpi_abi_version(void);
const char* gmpi_last_error(void);

/* Name of the kernel variant a forward call with these shapes would launch (diagnostics). */
const char* gmpi_mpi_render_fwd_variant(int N, int Ht, int Wt, int H, int W);

/*
 * Which FORWARD kernels a call with these shapes launches, for one fp32 MPI rgba [1,N,4,Ht,Wt]: GMPI_PLAN_STAGED (persistent
 * TMA-staged kernels, the fast path) or GMPI_PLAN_DIRECT (one thread per pixel, any shape, several times slower).  *why (nullable)
 * receives the GMPI_WHY_* bits of every reason the staged path is not taken, so a caller can surface the performance cliff
 * instead of finding it in a profile.  rgba may be NULL (alignment unknown: not checked).  gmpi_mpi_render_fwd_plan_ex answers
 * for a whole descriptor (M MPIs, factored, fp16).  The early-stop and training forwards get the same plan as the plain one.  The
 * plan assumes the MPI's tensor maps encode; if cuTensorMapEncodeTiled refuses them, the forward takes the direct kernels (or
 * fails, under gmpi_debug_set_fwd_variant(2)).  The backward's kernel, and every reason it is not the staged one, comes from
 * gmpi_mpi_render_bwd_plan_ex (GMPI_WHY_NO_TRANSMITTANCE and up).
 */
#define GMPI_PLAN_DIRECT 1
#define GMPI_PLAN_STAGED 2
#define GMPI_WHY_TEX_WIDTH 1u    /* Wt % 4 != 0 (fp16: Wt % 8, uint8: Wt % 16): rows are not 16-byte multiples, no tensor map */
#define GMPI_WHY_FEW_TILES 2u    /* fewer than 120 tiles of 64x30 pixels over all views: the persistent grid would idle */
#define GMPI_WHY_MANY_PLANES 4u  /* N > 512: the per-view plane-constant table does not fit next to the ring, or
                                    M*N >= 2^31 planes over all MPIs                                                    */
#define GMPI_WHY_ALIGNMENT 8u    /* an MPI base (rgba, rgb, alpha or bg_rgb) not 16-byte aligned                        */
#define GMPI_WHY_FORCED 16u      /* gmpi_debug_set_fwd_variant(1)                                                        */
/* the backward's own reasons (gmpi_mpi_render_bwd_plan_ex) */
#define GMPI_WHY_NO_TRANSMITTANCE 32u   /* no saved transmittance: the forward did not save one for the box kernel's sweep       */
#define GMPI_WHY_IMG_WIDTH 64u          /* W % 4 != 0: the transmittance's rows are not 16-byte multiples, no tensor map         */
#define GMPI_WHY_GRAD_ALIGNMENT 128u    /* a gradient base (g_rgba, or g_rgb, g_alpha, g_bg_rgb) or the transmittance base is
                                           not 16-byte aligned                                                                 */
#define GMPI_WHY_MANY_PIXEL_PLANES 256u /* V*N >= 2^31 pixel planes of transmittance                                            */
int gmpi_mpi_render_fwd_plan(int V, int N, int Ht, int Wt, int H, int W, const void* rgba, uint32_t* why);

/*
 * Forward: replaces MPI.forward (mpi.py:308-436) for all V views in one launch.
 * Per output pixel the planes are walked front to back; colour, depth and transmittance stay in
 * registers; no [V*N, c, H, W] intermediate is written.
 * Numerics: texel coordinates are bit-identical to the reference's fp32 op sequence.  The transmittance is updated as
 * T <- T - a*T in the TMA-staged kernels and as T <- T*((1-a)+1e-10) (the reference's form, mpi.py:421) in the direct kernels:
 * the two differ by < 1e-10 absolute per plane, far below the fp32 resolution of the outputs; both are within 1e-6 (relative
 * to the largest output) of the reference, and so is the transmittance saved for the backward.  Up to 65535 views per launch
 * on the direct kernels (gmpi_mpi_render_fwd_plan tells which kernel a shape gets); the staged kernels have no such limit.
 */
int gmpi_mpi_render_fwd(const float* rgba, const int32_t* view2mpi, const float* dhw,
                        const float* ray_dir, const float* eye, const float* z_dir,
                        float* color, float* depth, uint32_t* flags,
                        int M, int V, int N, int Ht, int Wt, int H, int W,
                        uint32_t options, void* stream);

/*
 * Forward with the all-gather of frames fused into the epilogue (multi-GPU, SURVEY.md section 8e).  Instead of
 * color/depth, every finished pixel of view v is stored as a packed frame [4,H,W] = (R,G,B,depth) at frame index
 * frame_offset + v of EVERY buffer in peer_frames: a DEVICE array of n_peers base pointers to [F,4,H,W] fp32 buffers,
 * one per rank, peer-mapped over NVLink (e.g. torch symmetric memory, cudaIpc).  The stores are posted writes that overlap
 * the remaining compute; the caller makes them visible with a barrier across ranks after the kernel.  Replaces the
 * render + ncclAllGather pair; the reference has no counterpart (its renderer is single-GPU, gloo barriers only).
 * Preconditions the library cannot check, because the pointer array is in device memory:
 *   - every peer_frames[r] base is 16-byte aligned (the epilogue stores float4s when W % 4 == 0);
 *   - every buffer holds F >= frame_offset + V frames.
 */
int gmpi_mpi_render_fwd_gather(const float* rgba, const int32_t* view2mpi, const float* dhw,
                               const float* ray_dir, const float* eye, const float* z_dir,
                               float* const* peer_frames, int n_peers, int frame_offset, uint32_t* flags,
                               int M, int V, int N, int Ht, int Wt, int H, int W,
                               uint32_t options, void* stream);

/*
 * Backward: d(sum(color*g_color) + sum(depth*g_depth)) / d rgba, what torch autograd produces for
 * MPI.forward (only the sampled rgba carries gradient: mpi.py:65,148 run under no_grad).
 * g_depth may be NULL.  Views of one MPI accumulate into the same g_rgba slab (the `expand` of
 * train.py:733-738).  g_rgba must be zero, or pass GMPI_ZERO_GRAD.
 * If options has GMPI_COLOR_MINUS1_1 the upstream g_color is w.r.t. 2*color-1.
 */
int gmpi_mpi_render_bwd(const float* rgba, const int32_t* view2mpi, const float* dhw,
                        const float* ray_dir, const float* eye, const float* z_dir,
                        const float* g_color, const float* g_depth, float* g_rgba,
                        int M, int V, int N, int Ht, int Wt, int H, int W,
                        uint32_t options, void* stream);

/*
 * Training pair.  gmpi_mpi_render_fwd_train = gmpi_mpi_render_fwd that additionally saves the transmittance in front of
 * every plane, transmittance [V,N,H,W] (T_i = prod_{j<i}(1 - alpha_j), mpi.py:421-423) -- what torch autograd keeps alive as
 * `weights`/`cumprod` tensors, here 4 bytes per (pixel, plane).  gmpi_mpi_render_bwd_saved consumes it: one staged
 * back-to-front sweep instead of the two-pass kernel, where gmpi_mpi_render_bwd_plan_ex of the same call answers
 * GMPI_PLAN_STAGED; otherwise the call runs gmpi_mpi_render_bwd's two-pass kernel.
 */
int gmpi_mpi_render_fwd_train(const float* rgba, const int32_t* view2mpi, const float* dhw,
                              const float* ray_dir, const float* eye, const float* z_dir,
                              float* color, float* depth, float* transmittance, uint32_t* flags,
                              int M, int V, int N, int Ht, int Wt, int H, int W,
                              uint32_t options, void* stream);
int gmpi_mpi_render_bwd_saved(const float* rgba, const int32_t* view2mpi, const float* dhw,
                              const float* ray_dir, const float* eye, const float* z_dir,
                              const float* transmittance, const float* g_color, const float* g_depth,
                              float* g_rgba, int M, int V, int N, int Ht, int Wt, int H, int W,
                              uint32_t options, void* stream);

/*
 * Descriptor form of the render calls: every optional input/output of the path in one struct, so that the variants below
 * compose (factored MPI x in-kernel rays x video epilogue x fused all-gather x training).  Zero-initialise it, set
 * struct_bytes = sizeof(gmpi_render_desc) and fill what applies; every pointer is DEVICE memory for gmpi_mpi_render_fwd_ex /
 * gmpi_mpi_render_bwd_ex and HOST memory for gmpi_mpi_render_host_ex.
 *
 *   MPI, one of
 *     rgba   [M,N,4,Ht,Wt]                       the expanded stack MPI.forward receives (mpi.py:309)
 *     rgb    [M,3,Ht,Wt] + alpha [M,N,1,Ht,Wt]   the generator's FACTORED output: one colour image shared by all planes and one
 *            (+ bg_rgb [M,3,Ht,Wt], optional)    alpha per plane, before the reference expands and concatenates them
 *                                                (networks_cond_on_pos_enc.py:950-975,984,1313; bg_rgb = the last plane's own
 *                                                colour under torgba_sep_background).  4x fewer HBM / PCIe bytes; output
 *                                                identical to rendering the expanded stack.
 *   camera, one of
 *     ray_dir [V,3,H,W] + eye [V,3] + z_dir [V,3]   the reference's tensors (parity mode: bit-exact texel coordinates)
 *     cam [V,16] = {f0, f1, f2 (the fp64 focal length as three fp32 pieces with f0 + f1 + f2 == focal exactly), pixel-centre
 *                   offset (0.5), R row-major (9), eye (3)}; the principal point is (W/2, H/2) (cam_utils.py:20)
 *                                                fast mode: rays generated in the kernel with camera.py:53-118,182-211's
 *                                                arithmetic (fp64 camera ray -> fp32 -> fp32 rotation); saves the [V,3,H,W]
 *                                                tensor and its upload.  Forward only.
 *   view_group  > 1 when every view_group consecutive views share one MPI (V % view_group == 0): tiles are then ordered so that
 *               concurrently running CTAs work on the same texels (L2 reuse; video render, multi-view search).  0/1 otherwise.
 *   outputs, one of
 *     color [V,3,H,W] + depth [V,1,H,W]          fp32 (2c-1 with GMPI_COLOR_MINUS1_1)
 *     peer_frames / n_peers / frame_offset       fused all-gather, see gmpi_mpi_render_fwd_gather.  A single NVLS multicast
 *                                                address with n_peers = 1 makes the switch replicate the stores.
 *     video_rgb [V,H,W,3] uint8 + video_depth [V,H,W,1] uint8 (optional), depth_near / depth_range
 *                                                the conversion lines of render_video.py:118-126 fused into the store:
 *                                                ((2c-1)+1)/2*255 truncated; clip((d - near)/range, 0, 1)*255 truncated
 *                                                (GMPI_U8_ROUND_HALF_UP: torchvision save_image rounding instead)
 *   transmittance [V,N,H,W]                      training forward: saved for gmpi_mpi_render_bwd_ex
 *   backward: g_color [V,3,H,W], g_depth (nullable), and g_rgba [M,N,4,Ht,Wt]  or  g_rgb [M,3,Ht,Wt] (+ g_bg_rgb) + g_alpha
 *             [M,N,1,Ht,Wt]; zeroed by the callee with GMPI_ZERO_GRAD, else accumulated into
 */
typedef struct gmpi_render_desc {
    uint32_t struct_bytes;
    uint32_t options;
    int32_t M, V, N, Ht, Wt, H, W;
    int32_t view_group;
    int32_t n_peers, frame_offset;
    float depth_near, depth_range;
    const float* rgba;
    const float* rgb;
    const float* alpha;
    const float* bg_rgb;
    const int32_t* view2mpi;
    const float* dhw;
    const float* ray_dir;
    const float* eye;
    const float* z_dir;
    const float* cam;
    float* color;
    float* depth;
    float* transmittance;
    float* const* peer_frames;
    uint8_t* video_rgb;
    uint8_t* video_depth;
    const float* g_color;
    const float* g_depth;
    float* g_rgba;
    float* g_rgb;
    float* g_bg_rgb;
    float* g_alpha;
    uint32_t* flags;
    void* stream;
    float early_stop;
} gmpi_render_desc;

/*
 * early_stop (with GMPI_EARLY_STOP in options; off by default): a threshold 0 <= tau < 1.  After plane i is composited, a pixel
 * whose transmittance satisfies |T| <= tau composites no further plane; its colour and depth are what it accumulated so far.  The
 * planes dropped carry a total weight of at most T <= tau, so each colour channel moves by at most tau (2 tau with
 * GMPI_COLOR_MINUS1_1), depth by at most tau * (the pixel's largest z-depth over the planes) and a uint8 output by at most one
 * code.  tau = 0 gives bit-identical output to early stop off.  The decision is per pixel, so the output does not depend on
 * timing.  The staged kernels skip the plane loads of a tile once all its pixels have stopped.  Forward only: a descriptor that
 * also sets transmittance, and every backward call with the bit, return GMPI_ERR_UNSUPPORTED.  The classic entry points have no
 * threshold field and refuse the bit.
 *
 * struct_bytes: sizeof(gmpi_render_desc), or GMPI_RENDER_DESC_V2_BYTES, the size before early_stop was appended (callers built
 * against that header keep working; early stop is then off and GMPI_EARLY_STOP is refused).
 */
#define GMPI_RENDER_DESC_V2_BYTES offsetof(gmpi_render_desc, early_stop)

/*
 * GMPI_MPI_F16 (off by default): every MPI tensor of the call -- rgba, or rgb + alpha (+ bg_rgb) -- is IEEE binary16, with the
 * layouts above; the descriptor's float pointers are read as pointers to halves.  Every other input and every output keeps its type.
 * An fp16 value converts to fp32 exactly and the kernels convert each texel tap before the unchanged fp32 arithmetic, so the output
 * is bitwise equal to the same call on the fp32 upcast of the MPI (on the same kernel variant and ring depth), at half the MPI bytes
 * read from HBM -- and, through gmpi_mpi_render_host_ex, uploaded.  The staged kernels need Wt % 8 == 0 and 16-byte aligned MPI
 * bases (gmpi_mpi_render_fwd_plan_ex); other shapes take the direct kernels.  Accepted by gmpi_mpi_render_fwd_ex,
 * gmpi_mpi_render_fwd_skip_ex, gmpi_mpi_render_host_ex, gmpi_mpi_render_fwd_plan_ex, gmpi_mpi_occupancy_bytes and
 * gmpi_mpi_build_occupancy.  GMPI_ERR_UNSUPPORTED for a descriptor that sets transmittance, the backward calls and every classic
 * entry point.  The deterministic scratch query does not refuse the bit (nor GMPI_EARLY_STOP): it returns the size, and the
 * deterministic backward refuses the call.
 *
 * GMPI_MPI_U8 (off by default): rgba is uint8 [M,N,4,Ht,Wt] (the planar layout of RGBA8 plane images after the reference's permute,
 * mpi_utils.py:336-337); the descriptor's rgba pointer is read as a pointer to bytes and code b stands for b / 255 rounded to nearest
 * in fp32.  The kernels convert each texel tap exactly before the unchanged fp32 arithmetic, so the output (colour, depth, uint8
 * frames, flags) is bitwise equal to the same call on the fp32 tensor rgba / 255 (on the same kernel variant and ring depth), at a
 * quarter of the fp32 MPI's bytes read from HBM -- and, through gmpi_mpi_render_host_ex, uploaded.  The staged kernels need
 * Wt % 16 == 0 and a 16-byte aligned rgba (gmpi_mpi_render_fwd_plan_ex); other shapes take the direct kernels.  Accepted by
 * gmpi_mpi_render_fwd_ex, gmpi_mpi_render_fwd_skip_ex, gmpi_mpi_render_host_ex, gmpi_mpi_render_fwd_plan_ex, gmpi_mpi_occupancy_bytes
 * and gmpi_mpi_build_occupancy; composes with GMPI_EARLY_STOP, cam, view_group, the video outputs and the fused gather.  Together
 * with GMPI_MPI_F16: GMPI_ERR_INVALID_ARGUMENT.  GMPI_ERR_UNSUPPORTED for a factored MPI (rgb / alpha / bg_rgb set), a descriptor
 * that sets transmittance, the backward calls, the deterministic scratch query and every classic entry point.
 */

/* cudaMemsetAsync(ptr, 0, bytes) on `stream`, for callers that accumulate into their own buffers (no GMPI_ZERO_GRAD).  Note that a
 * memset cannot overlap the staged kernels, on whatever stream (they own every SM: measured, tools/zero_overlap_probe.py). */
int gmpi_mpi_zero_async(void* ptr, size_t bytes, void* stream);

int gmpi_mpi_render_fwd_ex(const gmpi_render_desc* desc);
/* gmpi_mpi_render_fwd_plan for the forward a descriptor describes (sizes, options, MPI pointers; the other fields are not read):
 * the plan gmpi_mpi_render_fwd_ex launches with.  It sees GMPI_MPI_F16 and GMPI_MPI_U8: an fp16 MPI needs Wt % 8 == 0 and a
 * uint8 MPI Wt % 16 == 0 for the staged kernels (GMPI_WHY_TEX_WIDTH otherwise).  The MPI's pointers (rgba, or rgb + alpha + bg_rgb) must be 16-byte
 * aligned (GMPI_WHY_ALIGNMENT); NULL ones are not checked.  Forward only, like gmpi_mpi_render_fwd_plan.  Returns the plan, or a
 * negative GMPI_ERR_* code for a bad descriptor. */
int gmpi_mpi_render_fwd_plan_ex(const gmpi_render_desc* desc, uint32_t* why);
/* The backward kernel gmpi_mpi_render_bwd_ex and gmpi_mpi_render_bwd_deterministic_ex (which makes the same choice) launch for a
 * descriptor, asked before the training forward runs: GMPI_PLAN_STAGED (the box kernel, one back-to-front sweep over the saved
 * transmittance) or GMPI_PLAN_DIRECT (the two-pass kernel, which walks every plane twice).  *why (nullable) receives the GMPI_WHY_*
 * bits of every reason it is not the box kernel: those of gmpi_mpi_render_fwd_plan_ex for the same descriptor (the box kernel reads
 * the MPI as the staged forward does), and GMPI_WHY_NO_TRANSMITTANCE (transmittance NULL), GMPI_WHY_IMG_WIDTH,
 * GMPI_WHY_GRAD_ALIGNMENT and GMPI_WHY_MANY_PIXEL_PLANES.  It reads the sizes, the options, view_group, cam, the MPI pointers, the
 * gradient pointers and the transmittance pointer, and nothing else; no pointer need be set, and NULL MPI and gradient pointers count
 * as aligned.  It needs no GPU.  It refuses what the backward calls refuse before launching, with the same negative GMPI_ERR_* code
 * and gmpi_last_error() text, except that it asks for no pointer: the forward-only options (GMPI_MPI_F16, GMPI_MPI_U8,
 * GMPI_EARLY_STOP), cam, bad sizes or view_group, and the direct kernel's limits (more than 65535 views, too tall an image, more
 * planes than its stash holds) where it takes the direct kernel with V > 0; on that last refusal *why is still written.  It assumes the
 * tensor maps encode, as gmpi_mpi_render_fwd_plan_ex does.  The deterministic backward's own refusals (its scratch, and shapes that
 * leave fewer than 24 fraction bits) are not the plan's. */
int gmpi_mpi_render_bwd_plan_ex(const gmpi_render_desc* desc, uint32_t* why);
int gmpi_mpi_render_bwd_ex(const gmpi_render_desc* desc);

/*
 * Deterministic backward (opt-in): gmpi_mpi_render_bwd_ex with bitwise-reproducible gradients.  The same inputs give the same bits
 * on every call, and so do the views of an MPI permuted together with their rays and upstream gradients.  It takes the same
 * descriptors and kernel choice as gmpi_mpi_render_bwd_ex (the staged box kernel with a saved transmittance where that call would
 * use it, the direct kernel otherwise) and refuses what that call refuses.  Every contribution is rounded to a per-call unit
 * 2^(E - k) and summed exactly in int64 (red.global.add.u64) in `scratch`, so the order of the hardware's additions does not matter:
 *   E  from the largest upstream gradient of the call (a pre-pass over every pixel of every view; inf/NaN left out), clamped to
 *      [-100, 128];
 *   k  = 61 - ceil(log2(H*W)) - ceil(log2(V)) - ceil(log2(planes summed into one element: N for a factored MPI's colour, else 1)),
 *      so that no element's sum can wrap (GMPI_ERR_UNSUPPORTED below 24 bits).
 * Each gradient is within (contributions) * 2^(E-k-1) + 2^-24 |gradient| of the exact sum of its contributions, on top of the
 * staged kernel's per-tile fixed point that gmpi_mpi_render_bwd_ex has too (DESIGN.md section 4.3).  An inf/NaN contribution gives
 * what an fp32 sum gives: NaN if a NaN or both infinities were added, else that infinity.  Results written with GMPI_ZERO_GRAD,
 * added into the gradient buffers without it.
 * scratch: device memory of at least gmpi_mpi_render_bwd_deterministic_scratch_bytes(desc) bytes, 16-byte aligned; zeroed by the
 * callee on the stream; 8 bytes per gradient element plus half a byte of non-finite bits plus 256.  The callee allocates nothing.
 * The scratch-size query reads the sizes and which MPI pointers (rgba, or rgb + alpha with or without bg_rgb) are set; it
 * returns the bytes, or a negative GMPI_ERR_* code.  Neither needs a GPU to refuse a call.
 */
long long gmpi_mpi_render_bwd_deterministic_scratch_bytes(const gmpi_render_desc* desc);
int gmpi_mpi_render_bwd_deterministic_ex(const gmpi_render_desc* desc, void* scratch, size_t scratch_bytes);

/*
 * Opt-in empty-space skipping (forward only).  A texel of plane i of MPI m is EMPTY when its alpha is +0.0 (bit pattern 0; -0.0 and
 * NaN count as occupied) and its three colour values are finite (factored MPI: the shared rgb texel, or bg_rgb's on the last plane).
 * The occupancy map holds one bit per 8 x 8 texel block of every (MPI, plane), set when a texel of the block is not empty: per plane
 * ceil(Ht/8) rows of ceil(ceil(Wt/8)/32) 32-bit words, bit b of word w = block column 32 w + b; planes in the order m * N + i.
 *
 * gmpi_mpi_occupancy_bytes: the map's size for desc (its sizes and MPI pointers: rgba, or rgb + alpha), or a negative GMPI_ERR_*.
 * gmpi_mpi_build_occupancy: fills the map (device memory, 4-byte aligned, at least the size above) from desc's MPI (fp32, fp16
 *   under GMPI_MPI_F16, or uint8 under GMPI_MPI_U8: empty iff the alpha byte is 0) on desc->stream.  For an fp32 or fp16 expanded
 *   MPI with desc->flags set it also ORs in the GMPI_FLAG_RGBA_RANGE | GMPI_FLAG_ALPHA_RANGE bits that gmpi_mpi_check_range(_f16)
 *   would set, from the same pass (a uint8 MPI is always inside [0, 1]: its build does not read the flags).
 * gmpi_mpi_render_fwd_skip_ex: gmpi_mpi_render_fwd_ex, except that the TMA-staged forward arms a (tile, plane) stage without
 *   loading it when every texel under its box is empty, and composites nothing where its taps fall in that box.  Compositing such a
 *   box adds fma(+0, finite, x) == x to colour and depth and leaves T alone, so colour, depth, uint8 frames and flags are bitwise
 *   those of gmpi_mpi_render_fwd_ex whenever no accumulator is -0.0 and T is finite in front of a skipped stage (DESIGN.md section
 *   4.1: true for every MPI inside the range check's [0, 1]).  The direct kernel takes the request and skips nothing.  Composes with
 *   the factored MPI, GMPI_MPI_F16, GMPI_MPI_U8, GMPI_EARLY_STOP, cam, view_group, the video outputs and the fused gather; refuses a
 *   descriptor with transmittance and a map smaller than gmpi_mpi_occupancy_bytes.  The map must describe the MPI as it is now: the callee
 *   cannot tell a stale map.  None of the three needs a GPU to refuse a call.
 */
long long gmpi_mpi_occupancy_bytes(const gmpi_render_desc* desc);
int gmpi_mpi_build_occupancy(const gmpi_render_desc* desc, void* occ, size_t bytes);
int gmpi_mpi_render_fwd_skip_ex(const gmpi_render_desc* desc, const void* occ, size_t bytes);

/* Host-buffer form (end-to-end entry point, see gmpi_mpi_render_fwd_host): all pointers of *desc are HOST memory, `stream` is
 * ignored, *flags receives the flag word.  Forward only; supports the factored MPI, cam and the video outputs. */
int gmpi_mpi_render_host_ex(const gmpi_render_desc* desc, int device);

/*
 * LightRenderer (gmpi/core/light_renderer.py), the lighting augmentation applied to the MPI right before the render call in
 * training (train.py:534-541,702-709).  Two streaming kernels replace what the reference materialises:
 *
 * gmpi_mpi_alpha_depth_fwd = LightRenderer.compute_depth (light_renderer.py:82-100): the over-composite of the UN-warped alpha,
 *   depth[m] = sum_i a_i prod_{j<i}(1 - a_j + 1e-10) plane_d[i]  -> depth [M,1,Ht,Wt].  alpha of plane i of MPI m is read at
 *   alpha[m * mpi_stride + i * plane_stride + texel] (strides in floats): the expanded stack (alpha = rgba + 3*Ht*Wt, plane_stride
 *   = 4*Ht*Wt, mpi_stride = N*4*Ht*Wt) or the factored alpha [M,N,1,Ht,Wt] (plane_stride = Ht*Wt).  transmittance [M,N,Ht,Wt] is
 *   optional (training: saved for the backward).  gmpi_mpi_alpha_depth_bwd: d sum(depth * g_depth) / d alpha into g_alpha with its
 *   own strides (e.g. channel 3 of a g_rgba stack).
 * gmpi_mpi_apply_shading_fwd = the last step of LightRenderer.render (light_renderer.py:190-199): out[m,i,c] =
 *   clip(rgba[m,i,c] * shade[m], 0, 1) for the colour channels, alpha copied: the new [M,N,4,Ht,Wt] MPI in one pass.
 *   _bwd: gradients w.r.t. rgba and shade [M,1,Ht,Wt] (torch.clip's closed-interval mask).
 */
int gmpi_mpi_alpha_depth_fwd(const float* alpha, long long mpi_stride, long long plane_stride, const float* plane_d,
                             float* depth, float* transmittance, int M, int N, int Ht, int Wt, void* stream);
int gmpi_mpi_alpha_depth_bwd(const float* alpha, long long mpi_stride, long long plane_stride, const float* plane_d,
                             const float* transmittance, const float* g_depth, float* g_alpha, long long g_mpi_stride,
                             long long g_plane_stride, int M, int N, int Ht, int Wt, void* stream);
int gmpi_mpi_apply_shading_fwd(const float* rgba, const float* shade, float* out, int M, int N, int Ht, int Wt, void* stream);
int gmpi_mpi_apply_shading_bwd(const float* rgba, const float* shade, const float* g_out, float* g_rgba, float* g_shade,
                               int M, int N, int Ht, int Wt, void* stream);

/*
 * Range checks of MPIRenderer.render (mpi_renderer.py:447-449) and MPI.check_shapes
 * (mpi.py:185-187) in one streaming pass: sets GMPI_FLAG_RGBA_RANGE / GMPI_FLAG_ALPHA_RANGE.
 */
int gmpi_mpi_check_range(const float* rgba, int M, int N, int Ht, int Wt, uint32_t* flags,
                         void* stream);
/* The same check of an fp16 rgba [M,N,4,Ht,Wt]: sets the flags gmpi_mpi_check_range sets on its fp32 upcast (NaN included). */
int gmpi_mpi_check_range_f16(const void* rgba, int M, int N, int Ht, int Wt, uint32_t* flags, void* stream);

/*
 * Host-buffer forward (end-to-end entry point): all pointers are HOST memory (pinned memory
 * overlaps best).  Copies inputs to `device`, renders, copies colour/depth/flags back and
 * synchronises.  MPIs are streamed through a double-buffered device staging area so the copy of
 * MPI m+1 overlaps the render of MPI m.  *flags_out receives the OR of all flag bits.  The staging buffers, streams and
 * events are cached per device (grow-only) across calls; gmpi_mpi_release_host_cache() frees them.
 */
int gmpi_mpi_render_fwd_host(const float* rgba, const int32_t* view2mpi, const float* dhw,
                             const float* ray_dir, const float* eye, const float* z_dir,
                             float* color, float* depth, uint32_t* flags_out,
                             int M, int V, int N, int Ht, int Wt, int H, int W,
                             uint32_t options, int device);

int gmpi_mpi_release_host_cache(void);

/* Test hook: texel coordinates (ix, iy) of every (view, plane, pixel), out [V,N,2,H,W]; the
 * bit-exact stage of the path (must equal torch's fp32 op sequence, DESIGN.md "coordinates"). */
int gmpi_debug_plane_coords(const int32_t* view2mpi, const float* dhw, const float* ray_dir,
                            const float* eye, float* out, int V, int N, int Ht, int Wt, int H,
                            int W, uint32_t options, void* stream);

/* Test hook: same as gmpi_debug_plane_coords through the staged kernel's pixel-pair coordinate code (H*W even). */
int gmpi_debug_plane_coords_packed(const int32_t* view2mpi, const float* dhw, const float* ray_dir,
                                   const float* eye, float* out, int V, int N, int Ht, int Wt, int H,
                                   int W, uint32_t options, void* stream);

/* Test hook: force the forward kernel variant: 0 auto (default), 1 direct-gather, 2 TMA-staged. */
int gmpi_debug_set_fwd_variant(int variant);

/* Test hook: force the ring depth of the expanded TMA-staged forward: 0 auto (default), 2 or 3 stages.  The factored forward
 * keeps its 3-stage ring. */
int gmpi_debug_set_fwd_stages(int stages);

/* Test hook: the last GMPI_EARLY_STOP launch on this device (synchronises the device): *skipped = the (tile, plane) stages the
 * staged kernel armed without loading their box, *total = the stages it walked (tiles x N; 0 when the direct kernel ran). */
int gmpi_debug_fwd_early_stop_stats(unsigned long long* skipped, unsigned long long* total);

/* Test hook: the last gmpi_mpi_render_fwd_skip_ex launch on this device (synchronises the device): *skipped = the (tile, plane)
 * stages the staged kernel armed empty, *total = the stages it walked (0 when the direct kernel ran). */
int gmpi_debug_fwd_skip_stats(unsigned long long* skipped, unsigned long long* total);

/* Test hook (host only, does not synchronise): *key = the variant key (the kKey* bits of csrc/mpi_kernel_keys.cuh) of the last render
 * kernel, forward or backward, the library launched on `device` from any thread; GMPI_ERR_INVALID_ARGUMENT before the first. */
int gmpi_debug_last_render_key(int device, uint32_t* key);

/* Test hook (host only): the staged producer's box-versus-map test on one plane's map (host memory, the layout of
 * gmpi_mpi_build_occupancy): 1 when a block under the texels [bx0, bx0 + bw) x [by0, by0 + rows) inside the Ht x Wt texture is
 * occupied, 0 when the box is empty, a negative GMPI_ERR_* code on bad arguments. */
int gmpi_debug_box_occupied(const uint32_t* plane_map, int Ht, int Wt, int bx0, int by0, int bw, int rows);

/* Test hooks of the GMPI_MPI_U8 conversion: out[b] = the fp32 value of code b for the 256 codes.  _host: the host build, out is host
 * memory (no GPU work); without the suffix: the device build (a kernel of mpi_u8.cu), out is device memory, on `stream`. */
int gmpi_debug_u8_codes_host(float* out);
int gmpi_debug_u8_codes(float* out, void* stream);

/* Test hook: the ring depth (2 or 3) the expanded staged forward picks on the current device for M MPIs, V views, N planes of
 * Ht x Wt texels and view_group (gmpi_render_desc.view_group); a negative GMPI_ERR_* code on bad arguments. */
int gmpi_debug_fwd_ring_stages(int M, int V, int N, int Ht, int Wt, int view_group);

/* Test hook (host only): the TMA copies the expanded forward issues for a footprint of n_rows staged rows, as (first row, rows)
 * pairs: the binary digits of n_rows / 4 (copies of 32, 16, 8, 4 rows).  Returns the number of copies. */
int gmpi_debug_copy_plan(int n_rows, int* out_row_rows, int max_copies);

/* Test hook (host only): tile order for a tile height (30 forward, 24 backward) and view grouping (gmpi_render_desc.view_group). */
int gmpi_debug_tile_walk_ex(int H, int W, int V, int tile_h, int view_group, int grid, int cta, int* out_v_px0_py0, int max_tiles);

/* Test hook: the rays the fast mode generates from cam [V,16] -> ray_dir [V,3,H,W] (device memory). */
int gmpi_debug_cam_rays(const float* cam, float* ray_dir, int V, int H, int W, void* stream);

/* Test hook (host only, no GPU work): the persistent kernels' tile order.  Writes the (view, px0, py0) of the tiles that
 * CTA `cta` of a `grid`-CTA launch walks, in order, into out_v_px0_py0[3 * max_tiles]; returns their number (>= 0) or a
 * negative GMPI_ERR_* code.  Tile size: 64 x 30 pixels. */
int gmpi_debug_tile_walk(int H, int W, int V, int grid, int cta, int* out_v_px0_py0, int max_tiles);

/* Test hook: out_fast[i] = the kernels' reciprocal+FMA division a[i]/b[i]; out_ieee[i] = div.rn.f32. */
int gmpi_debug_division(const float* a, const float* b, float* out_fast, float* out_ieee, size_t n,
                        void* stream);

#ifdef __cplusplus
}
#endif
#endif /* GMPI_MPI_RENDER_H_ */
