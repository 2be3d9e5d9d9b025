/* cspn_b200 -- C ABI of the H100-native CSPN propagation path.
 *
 * The reference (XinJCheng/CSPN) has no FFI: its hot path is a Python nn.Module,
 *   Affinity_Propagate.forward(guidance, blur_depth, sparse_depth=None)
 *     /root/reference/cspn_pytorch/models/cspn.py:42-83        (2D, 8 neighbours)
 *   fluid.layers.affinity_propagate(feat, gate_weight, kernel_size=3) iterated prop_step times
 *     /root/reference/cspn_paddle/demo.py:20-54                 (3D, 26 neighbours; op source not in tree)
 * Each entry point below is what a binding for those two call sites would bind
 * (INTEGRATION.md shows the ctypes stub and the drop-in `cspn.py`).
 *
 * Conventions
 *   - all tensors fp32, row-major NCHW / NCDHW, W fastest, dense (contiguous) planes;
 *   - *_f32 entry points take DEVICE pointers and enqueue on `stream` without synchronising
 *     or allocating; the caller provides `workspace` (size from *_workspace_bytes; may be
 *     NULL when that returns 0);
 *   - *_f32_host entry points take HOST pointers (pinned for full speed, pageable works),
 *     copy H2D / run / copy D2H in a chunked 3-stage pipeline and block until `out` is valid;
 *   - return value: CSPN_OK (0) or a negative cspn_status; cspn_last_error() gives the text
 *     (thread-local);
 *   - re-entrant and thread-safe: per-call state only, the tensor-map/launch-config cache is
 *     mutex-protected; one process per GPU is the intended deployment (torchrun), but
 *     DataParallel-style threads (reference eval.py:117) are safe too: the device of
 *     `blur`/`feat` is made current for the call and restored afterwards.
 */
#ifndef CSPN_B200_H_
#define CSPN_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct CUstream_st* cspn_stream_t; /* == cudaStream_t */

#if defined(__GNUC__)
#define CSPN_API __attribute__((visibility("default")))
#else
#define CSPN_API
#endif

typedef enum {
    CSPN_OK = 0,
    CSPN_ERR_INVALID_ARGUMENT = -1, /* bad shape / null pointer / unknown enum (reference: AssertionError, cspn.py:33,36) */
    CSPN_ERR_WORKSPACE = -2,        /* workspace missing or too small */
    CSPN_ERR_CUDA = -3,             /* a CUDA call failed; text in cspn_last_error() */
    CSPN_ERR_UNSUPPORTED = -4       /* requested algorithm cannot run this shape */
} cspn_status;

/* norm_type of Affinity_Propagate.__init__ (cspn.py:16-36) */
typedef enum {
    CSPN_NORM_8SUM = 0,     /* '8sum'     */
    CSPN_NORM_8SUM_ABS = 1  /* '8sum_abs' */
} cspn_norm2d;

/* 3D normalisation (SURVEY.md Appendix A.3) */
typedef enum {
    CSPN_NORM_26SUM = 0,     /* gathered affinities, signed, centre term (cspn.py scheme in 3D)          */
    CSPN_NORM_26SUM_ABS = 1, /* same with |g|                                                           */
    CSPN_NORM_PADDLE = 2     /* |g| normalised at the voxel's own location, no centre term (demo.py:24,47-52) */
} cspn_norm3d;

typedef enum {
    CSPN_ALGO_AUTO = 0,    /* cluster kernel when the shape allows, else generic                         */
    CSPN_ALGO_GENERIC = 1, /* prep kernel + one stencil launch per iteration (any shape; needs workspace) */
    CSPN_ALGO_CLUSTER = 2  /* TMA-staged tiles, register-resident state for all iterations of a launch, DSMEM halo
                              exchange inside a thread-block cluster.  One launch for prop_time <~ 24-32; longer
                              runs are split into passes and then need a workspace of B*C*H*W floats          */
} cspn_algo;

/* ---- 2D: replaces Affinity_Propagate.forward (cspn.py:42-83) --------------------------------
 * guidance [B][guidance_channels>=8][H][W] (channels 0..7 used, cspn.py:91-98)
 * blur     [B][C][H][W]   (C>1: affinity shared across channels, cspn.py:70 via Conv3d)
 * sparse   [B][1][H][W] or NULL (only its sign is used, cspn.py:63-64)
 * out      [B][C][H][W]   must not alias the inputs
 * iters    prop_time >= 0 (0 copies blur to out, cspn.py:61,83)
 */
/* Workspace for `algo`.  CSPN_ALGO_AUTO assumes what the cluster kernel needs of its tensors -- W % 4 == 0 and 16-byte
 * aligned base pointers (every allocator's default) -- because the query cannot see the pointers; if a call then has to
 * take the generic path (misaligned views), cspn2d_fwd_f32 returns CSPN_ERR_WORKSPACE with a message naming
 * cspn2d_workspace_bytes(..., CSPN_ALGO_GENERIC) as the size to provide.  The workspace should be 16-byte aligned too:
 * a cluster plan of several passes keeps its intermediate result there with 16-byte stores, so it declines a misaligned
 * workspace -- CSPN_ALGO_AUTO then takes the generic path as above, CSPN_ALGO_CLUSTER and cspn2d_fwd_gather_f32 return
 * CSPN_ERR_UNSUPPORTED.  The generic path takes any 4-byte aligned workspace. */
CSPN_API size_t cspn2d_workspace_bytes(int B, int C, int H, int W, int iters, int algo);

CSPN_API int cspn2d_fwd_f32(const float* guidance, const float* blur, const float* sparse, float* out,
                   int B, int C, int H, int W, int guidance_channels, int iters, int norm_type,
                   int algo, void* workspace, size_t workspace_bytes, cspn_stream_t stream);

CSPN_API int cspn2d_fwd_f32_host(const float* guidance, const float* blur, const float* sparse, float* out,
                        int B, int C, int H, int W, int guidance_channels, int iters, int norm_type,
                        int algo, int device);

/* ---- 2D forward fused with the final gather of a data-parallel run -----------------------------------------------
 * The reference gathers the replicas' outputs with nn.DataParallel (eval.py:117); one process per GPU does it with an
 * all-gather AFTER the kernel.  Here the kernel's epilogue stores every result tile to `out` and, tile by tile while it
 * goes on computing, to each peer_out[i] (the same [B][C][H][W] block inside the gather buffers of the other GPUs: peer
 * pointers mapped over NVLink, e.g. from a CUDA symmetric-memory allocation) and / or to multicast_out (an NVLS multicast
 * address: one multimem.st, replicated to all GPUs by the switch).  n_peer 0..7, multicast_out may be NULL; all
 * destinations 16-byte aligned.  Cluster kernel only (CSPN_ERR_UNSUPPORTED otherwise); workspace as for
 * CSPN_ALGO_CLUSTER.  The caller orders the remote stores before their consumers (a barrier across ranks after the
 * kernel: stores to peers are visible system-wide at kernel completion). */
CSPN_API int cspn2d_fwd_gather_f32(const float* guidance, const float* blur, const float* sparse, float* out,
                          float* const* peer_out, int n_peer, float* multicast_out,
                          int B, int C, int H, int W, int guidance_channels, int iters, int norm_type,
                          void* workspace, size_t workspace_bytes, cspn_stream_t stream);

/* ---- 2D backward (adjoint of the above; reference: autograd through cspn.py:42-83, used by
 * train.py:198).  grad_guidance [B][guidance_channels][H][W] (channels >= 8 are zero-filled),
 * grad_blur [B][C][H][W].  Either may be NULL.  Needs the forward inputs again.  Workspace: 9*B*H*W + 2*iters*B*C*H*W
 * floats (0 for iters == 0), on the cluster route and off it alike. */
CSPN_API size_t cspn2d_bwd_workspace_bytes(int B, int C, int H, int W, int iters);

CSPN_API int cspn2d_bwd_f32(const float* guidance, const float* blur, const float* sparse, const float* grad_out,
                   float* grad_guidance, float* grad_blur,
                   int B, int C, int H, int W, int guidance_channels, int iters, int norm_type,
                   void* workspace, size_t workspace_bytes, cspn_stream_t stream);

/* ---- 2D with a K x K affinity kernel, K in {3, 5, 7} (K*K-1 = 8, 24, 48 neighbours) ----------------------------
 * cspn.py with its pad tuples generalised (DESIGN.md section 4.8): tap k enumerates (t, l) over [0,K)^2 in raster order
 * without the centre and reads the source at (dy, dx) = ((K-1)/2 - t, (K-1)/2 - l).
 * guidance [B][guidance_channels >= K*K-1][H][W] (channels 0..K*K-2 used, shared across the C channels of blur);
 * blur / sparse / out / grad_* and norm_type (cspn_norm2d: 0 signed, 1 abs) as in the 3x3 calls above.
 * K = 3 IS the 3x3 operator: the calls delegate to cspn2d_fwd_f32 (CSPN_ALGO_AUTO) / cspn2d_bwd_f32 and the workspace
 * queries return theirs.  Forward workspace B*K*K*H*W + B*C*H*W floats at K = 5 / 7, backward B*K*K*H*W +
 * 2*iters*B*C*H*W floats at every K (0 for iters == 0); the size does not depend on the device.
 * CSPN_ERR_INVALID_ARGUMENT for K not in {3, 5, 7}, guidance_channels < K*K-1, an unknown norm, iters < 0, a non-positive shape or a null guidance / blur / out
 * (grad_out in the backward; grad_guidance and grad_blur may be NULL). */
CSPN_API size_t cspn2d_k_workspace_bytes(int B, int C, int H, int W, int K, int iters);

CSPN_API int cspn2d_k_fwd_f32(const float* guidance, const float* blur, const float* sparse, float* out,
                     int B, int C, int H, int W, int guidance_channels, int K, int iters, int norm_type,
                     void* workspace, size_t workspace_bytes, cspn_stream_t stream);

CSPN_API size_t cspn2d_k_bwd_workspace_bytes(int B, int C, int H, int W, int K, int iters);

CSPN_API int cspn2d_k_bwd_f32(const float* guidance, const float* blur, const float* sparse, const float* grad_out,
                     float* grad_guidance, float* grad_blur, int B, int C, int H, int W,
                     int guidance_channels, int K, int iters, int norm_type,
                     void* workspace, size_t workspace_bytes, cspn_stream_t stream);

/* ---- fused gather of the K x K, 'paddle' and gates forwards (2D) ----------------------------------------------------
 * cspn2d_k_fwd_gather_f32, cspn2d_paddle_fwd_gather_f32 and cspn2d_gates_fwd_gather_f32 take the arguments of their plain
 * forward plus peer_out / n_peer / multicast_out after `out`, as cspn2d_fwd_gather_f32 does, and give `out` its bits.  The
 * last step of the forward also stores its result to each peer_out[i] (the same [B][C][H][W] block inside another GPU's
 * gather buffer, a peer pointer mapped over NVLink) and / or to multicast_out (an NVLS multicast address, one
 * multimem.st); intermediate steps stay local.  n_peer 0..7 with a non-null array when non-zero, every peer_out[i]
 * non-null, every peer_out[i] and multicast_out (may be NULL) 16-byte aligned, else CSPN_ERR_INVALID_ARGUMENT;
 * iters == 0 is CSPN_ERR_UNSUPPORTED.
 * Workspace as for the plain forward (its *_workspace_bytes), and cspn_last_launches() counts the same launches.
 * K = 3 in cspn2d_k_fwd_gather_f32 delegates to cspn2d_fwd_gather_f32 and so needs the cluster kernel
 * (CSPN_ERR_UNSUPPORTED for a shape it cannot take, e.g. W % 4 != 0); the 'paddle' and gates entries take any W for
 * K in {3, 5, 7}.  Per-channel gates are B*C images with C = 1, as in the plain calls: the output memory, and with it the
 * peer offsets, is the same.  The caller orders the remote stores before their consumers (a barrier across ranks after
 * the call). */
CSPN_API int cspn2d_k_fwd_gather_f32(const float* guidance, const float* blur, const float* sparse, float* out,
                            float* const* peer_out, int n_peer, float* multicast_out,
                            int B, int C, int H, int W, int guidance_channels, int K, int iters, int norm_type,
                            void* workspace, size_t workspace_bytes, cspn_stream_t stream);

/* ---- 2D keep-sparse mode, K in {3, 5, 7}: the sparse samples are kept in the output (DESIGN.md section 4.13) ---------
 * The replacement step of the CSPN paper, H <- (1 - m) H + m sparse with m = 1[sparse > 0], in place of the reference
 * module's m = sign(sparse) and "+ m * blur":
 *   m = 1[sparse > 0] (NaN, 0 and negative samples -> 0);  d = blur;
 *   each of iters steps:  e = (1 - s) blur + sum_k w_k shift_k(d),  d = (1 - m) e + m sparse
 * with w_k, s = sum_k w_k and the taps of the K x K calls above, IEEE as written (0 * NaN = NaN, 0 * inf = NaN).  sparse
 * [B][1][H][W] is shared by the C channels of blur; a NULL sparse gives the default mode's bits (the K x K and 3x3 calls
 * above).  Arguments, shapes and status codes as in cspn2d_k_fwd_f32 / cspn2d_k_bwd_f32; `algo` (cspn_algo) chooses the
 * 3x3 path as in cspn2d_fwd_f32 and is ignored for K = 5 / 7, where the CSPN_B200_FORCE_* hooks do not apply either.
 * Workspace: K = 3 cluster plans as cspn2d_workspace_bytes; the launch-per-step paths (3x3 generic, K = 5 / 7) and every
 * backward one B*C*H*W plane more than the default mode's (d0' = (1 - m) blur + m sparse).  CSPN_ALGO_AUTO reports
 * CSPN_ERR_WORKSPACE as cspn2d_fwd_f32 does when a problem it sized for the cluster kernel falls back to the generic path.
 * The gather entry takes peer_out / n_peer / multicast_out after `out` as cspn2d_k_fwd_gather_f32 does (K = 3 on the
 * cluster kernel's epilogue, CSPN_ERR_UNSUPPORTED for a shape it cannot take; K = 5 / 7 on the last step).
 * The backward writes grad_guidance [B][guidance_channels][H][W], grad_blur [B][C][H][W] and
 * grad_sparse [B][1][H][W] = m * sum_c Gc_c (Gc_c = sum_t lambda_{t+1,c}; the channels summed in order, no atomics); any
 * of the three may be NULL.  grad_sparse is zero for a NULL sparse or iters == 0.  CUDA device pointers only: there is no
 * host-buffer entry. */
CSPN_API size_t cspn2d_keep_workspace_bytes(int B, int C, int H, int W, int K, int iters, int algo);

CSPN_API int cspn2d_keep_fwd_f32(const float* guidance, const float* blur, const float* sparse, float* out,
                        int B, int C, int H, int W, int guidance_channels, int K, int iters, int norm_type,
                        int algo, void* workspace, size_t workspace_bytes, cspn_stream_t stream);

CSPN_API int cspn2d_keep_fwd_gather_f32(const float* guidance, const float* blur, const float* sparse, float* out,
                               float* const* peer_out, int n_peer, float* multicast_out,
                               int B, int C, int H, int W, int guidance_channels, int K, int iters, int norm_type,
                               void* workspace, size_t workspace_bytes, cspn_stream_t stream);

CSPN_API size_t cspn2d_keep_bwd_workspace_bytes(int B, int C, int H, int W, int K, int iters);

CSPN_API int cspn2d_keep_bwd_f32(const float* guidance, const float* blur, const float* sparse, const float* grad_out,
                        float* grad_guidance, float* grad_blur, float* grad_sparse, int B, int C, int H, int W,
                        int guidance_channels, int K, int iters, int norm_type,
                        void* workspace, size_t workspace_bytes, cspn_stream_t stream);

/* ---- 2D aggregation of the steps, K in {3, 5, 7}: CSPN++'s context-aware CSPN (DESIGN.md section 4.20) --------------
 * d_0 = blur and d_{t+1} the step of cspn2d_k_fwd_f32 (keep = 0; sparse may be NULL) or of cspn2d_keep_fwd_f32 (keep = 1;
 * a NULL sparse gives the keep = 0 bits), every K on the K x K kernels; then, for the steps s_0 < ... < s_{T-1}
 * (steps, a HOST array of T = n_steps ints >= 1, strictly increasing; N = s_{T-1} steps run)
 *   out[b][c](p) = sum_j step_weight[b][j](p) * d_{s_j}[b][c](p)
 * summed over j ascending from the first term, every product and sum rounded on its own.  step_weight [B][T][H][W] is
 * used as given (no |.|, no normalisation) and shared by the C channels; a zero weight does not hide a NaN or an infinite
 * iterate (0 * inf = NaN).  guidance, blur, sparse, out, guidance_channels and norm_type as in the K x K calls above.
 * The backward writes grad_guidance [B][guidance_channels][H][W] (zero-filled first, as cspn2d_k_bwd_f32 does),
 * grad_blur [B][C][H][W], grad_sparse [B][1][H][W] (keep mode with a sparse: m * sum_c Gc_c as in cspn2d_keep_bwd_f32;
 * zero otherwise) and grad_step_weight [B][T][H][W] = sum_c grad_out[b][c](p) * d_{s_j}[b][c](p), c ascending from the
 * first term; any of the four may be NULL.
 * Workspace (floats; the queries return bytes, 0 for invalid arguments): forward B*K*K*H*W + (2 + keep)*B*C*H*W,
 * backward B*K*K*H*W + (2N + 1 + keep)*B*C*H*W, neither dependent on the device.  Launches: forward 1 + N, backward
 * 2 + 2N + ceil(T / 64).  No atomics; the only memsets are those of the K x K backward.
 * CSPN_ERR_INVALID_ARGUMENT for a null guidance / blur / step_weight / out (grad_out in the backward), a non-positive
 * shape, K not in {3, 5, 7}, guidance_channels < K*K-1, an unknown norm, keep not 0 or 1, n_steps < 1, a null steps, steps
 * not strictly increasing or < 1, a pointer that is not 4-byte aligned, and an output (the workspace included) that
 * overlaps an input or another output; CSPN_ERR_UNSUPPORTED for B*C > 65535; CSPN_ERR_WORKSPACE for a missing or short
 * workspace.  All of these come before any device work. */
CSPN_API size_t cspn2d_agg_workspace_bytes(int B, int C, int H, int W, int K, const int* steps, int n_steps, int keep);

CSPN_API int cspn2d_agg_fwd_f32(const float* guidance, const float* blur, const float* sparse, const float* step_weight,
                       float* out, int B, int C, int H, int W, int guidance_channels, int K, const int* steps,
                       int n_steps, int norm_type, int keep, void* workspace, size_t workspace_bytes, cspn_stream_t stream);

CSPN_API size_t cspn2d_agg_bwd_workspace_bytes(int B, int C, int H, int W, int K, const int* steps, int n_steps, int keep);

CSPN_API int cspn2d_agg_bwd_f32(const float* guidance, const float* blur, const float* sparse, const float* step_weight,
                       const float* grad_out, float* grad_guidance, float* grad_blur, float* grad_sparse,
                       float* grad_step_weight, int B, int C, int H, int W, int guidance_channels, int K,
                       const int* steps, int n_steps, int norm_type, int keep, void* workspace, size_t workspace_bytes,
                       cspn_stream_t stream);

/* ---- 2D non-local propagation, K in {3, 5, 7}: NLSPN's (Park et al., ECCV 2020) (DESIGN.md section 4.21) ---------
 * feat [B][C][H][W] is h_0; offset [B][2T][H][W], T = K*K - 1, channel 2k the dy and 2k + 1 the dx of tap k; affinity
 * [B][T][H][W] the weights a_k, used as given and shared by the C channels; sparse [B][C][H][W] or NULL.  Tap k runs over
 * (i, j) in [0, K)^2 in raster order without the centre, base offset (i - R, j - R), R = (K - 1) / 2: torchvision's and
 * DCN's order, the reverse of the K x K calls' (R - t, R - l).  S(h, y, x) is torchvision's bilinear_interpolate: 0 when
 * y <= -1, y >= H, x <= -1 or x >= W, NaN for a NaN position, otherwise the four corners at floor(y), floor(x) and one past,
 * a corner outside the image contributing nothing and one inside weight * value even when its weight is 0.  Then
 *   h_{t+1}(p) = a_c S(h~_t, p) + sum_k a_k S(h~_t, p + base_k + (dy_k(p), dx_k(p))),  a_c = 1 - sum_k a_k,
 *   h~_t = (1 - m) h_t + m sparse with m = 1[sparse > 0] (h~_t = h_t without a sparse); out = h_N, not replaced.
 * One step is deform_conv2d(h~_t, offset with a zero centre, ones(C, 1, K, K), padding = R, mask = affinity with a_c at
 * the centre), groups = C; the backward gives that composition's autograd gradients (torchvision's: a corner of weight
 * exactly 0 takes no part in grad_feat, and the offsets' coordinate weight has no window test).  Every operation is
 * rounded on its own in the order of DESIGN.md section 4.21: taps, then steps and channels ascending in every sum.
 * The backward writes any of grad_feat [B][C][H][W], grad_offset [B][2T][H][W], grad_affinity [B][T][H][W] and
 * grad_sparse [B][C][H][W] (sum_t m lambda~_t; needs a sparse) that is not NULL, and skips the work only the NULL ones need.
 * iters = 0: the forward copies feat to out, the backward copies grad_out and zero-fills the others.
 * Workspace (bytes; the queries return 0 for invalid arguments): forward 4 * min(iters - 1, 2) * B*C*H*W (0 for
 * iters <= 1).  Backward, with P = B*C*H*W, n = B*H*W*T and each region rounded up to 256 bytes:
 *   4 * (2 * iters * P + 2 * P + B*H*W + 8 * n) + 8 * (B*(H + 1)*(W + 1) + 1) + the radix sort's scratch + 256,
 * the last 256 bytes leaving room to start the regions at a 256-byte boundary of a 4-byte aligned workspace,
 * which CUB sizes for the current device: cspn2d_nl_bwd_workspace_bytes needs the CUDA runtime and a device and answers
 * 0 without one.  Launches: forward iters; backward at most (iters - 1) + 4 + the sort's + iters + 1.  No floating-point
 * atomics (the radix sort counts with integer ones); the bits depend on the arguments only.
 * CSPN_ERR_INVALID_ARGUMENT for a null feat / offset / affinity / out (grad_out in the backward), a non-positive shape, K
 * not in {3, 5, 7}, iters < 0, a grad_sparse without a sparse, a pointer that is not 4-byte aligned, and an output (the
 * workspace included) that overlaps an input or another output; CSPN_ERR_UNSUPPORTED for H*W*T >= 2^31,
 * B*ceil(C/4) > 65535 or B*(H+1)*(W+1) >= 2^32 - 1; CSPN_ERR_WORKSPACE for a missing or short workspace.  All of these come
 * before any device work. */
CSPN_API size_t cspn2d_nl_workspace_bytes(int B, int C, int H, int W, int K, int iters);

CSPN_API int cspn2d_nl_fwd_f32(const float* feat, const float* offset, const float* affinity, const float* sparse,
                      float* out, int B, int C, int H, int W, int K, int iters, void* workspace,
                      size_t workspace_bytes, cspn_stream_t stream);

CSPN_API size_t cspn2d_nl_bwd_workspace_bytes(int B, int C, int H, int W, int K, int iters);

CSPN_API int cspn2d_nl_bwd_f32(const float* feat, const float* offset, const float* affinity, const float* sparse,
                      const float* grad_out, float* grad_feat, float* grad_offset, float* grad_affinity,
                      float* grad_sparse, int B, int C, int H, int W, int K, int iters, void* workspace,
                      size_t workspace_bytes, cspn_stream_t stream);

/* ---- 2D dilated propagation, K in {3, 5, 7}, dilation in [1, 4]: PENet's DA-CSPN++ (Hu et al., ICRA 2021) --------------
 * (DESIGN.md section 4.22).  kernel [B][K*K][H][W] holds the weights as given (no abs, no normalisation), shared by the C
 * channels: channel j = i*K + l weights d_t(p + dilation*(i - R, l - R)), R = (K - 1) / 2 (F.unfold's row order), and the
 * centre channel c = (K*K - 1) / 2 weights blur(p).  blur [B][C][H][W] is d_0; sparse and confidence [B][1][H][W] are s and m,
 * both or neither, used as given.  A read outside the image is 0.  iters steps of
 *   u_t(p) = w_c(p) d_0(p) + sum_{j != c} w_j(p) d_t(p + dilation*o_j),  d_{t+1} = m s + (1 - m) u_t  (d_{t+1} = u_t without samples)
 * and out = d_N.  Order of operations (DESIGN.md section 4.22): u starts from the rounded product w_c d_0 and adds the taps
 * j = K*K-1 down to 0 by FMA; m s, (1 - m), its product with u and the sum are each rounded on their own.
 * The backward writes any of grad_kernel [B][K*K][H][W], grad_blur [B][C][H][W], grad_sparse and grad_confidence
 * [B][1][H][W] that is not NULL (the last two need the samples) and skips the work only the NULL ones need: without
 * grad_kernel and grad_confidence it recomputes no iterate.  iters = 0: the forward copies blur to out, the backward copies
 * grad_out and zero-fills the others (cudaMemsetAsync).
 * Workspace (bytes, device-independent; the queries return 0 for invalid arguments): forward 4 * B*C*H*W for iters >= 2,
 * else 0; backward 4 * (2 * iters - 1) * B*C*H*W (lambda_0 .. lambda_{N-1} and d_1 .. d_{N-1}), 0 for iters = 0.
 * Launches: forward iters; backward at most (iters - 1) + iters + 1.  No atomics; the bits depend on the arguments only.
 * CSPN_ERR_INVALID_ARGUMENT for a null kernel / blur / out (grad_out in the backward), exactly one of sparse and confidence,
 * a grad_sparse or grad_confidence without the samples, a non-positive shape, K not in {3, 5, 7}, a dilation outside
 * [1, 4], iters < 0, a pointer that is not 4-byte aligned, and an output (the workspace included) that overlaps an input
 * or another output; CSPN_ERR_UNSUPPORTED for B*C > 65535 or ceil(H/16) > 65535; CSPN_ERR_WORKSPACE for a missing or
 * short workspace.  All of these come before any device work. */
CSPN_API size_t cspn2d_dil_workspace_bytes(int B, int C, int H, int W, int K, int dilation, int iters);

CSPN_API int cspn2d_dil_fwd_f32(const float* kernel, const float* blur, const float* sparse, const float* confidence,
                       float* out, int B, int C, int H, int W, int K, int dilation, int iters, void* workspace,
                       size_t workspace_bytes, cspn_stream_t stream);

CSPN_API size_t cspn2d_dil_bwd_workspace_bytes(int B, int C, int H, int W, int K, int dilation, int iters);

CSPN_API int cspn2d_dil_bwd_f32(const float* kernel, const float* blur, const float* sparse, const float* confidence,
                       const float* grad_out, float* grad_kernel, float* grad_blur, float* grad_sparse,
                       float* grad_confidence, int B, int C, int H, int W, int K, int dilation, int iters,
                       void* workspace, size_t workspace_bytes, cspn_stream_t stream);

/* ---- 2D dynamic propagation, K in {3, 5, 7}: DySPN's step (Lin et al., AAAI 2022; DESIGN.md section 4.23) ---------------
 * affinity [B][K*K][H][W] holds all K*K taps, the centre included, as given (no abs, no normalisation), shared by the C
 * channels: channel j = i*K + l weights d_t(p + o_j), o_j = (i - R, l - R), R = (K - 1) / 2 (F.unfold's row order).  Tap j
 * lies on ring(j) = max(|i - R|, |l - R|).  attention [B][iters*(R+1)][H][W] holds, in channel t*(R+1) + r, the attention
 * of ring r at step t, as given.  blur [B][C][H][W] is d_0; sparse and confidence [B][1][H][W] are s and m, both or neither.
 * A read outside the image is 0.  iters steps of
 *   w_j = a_{t,ring(j)} affinity_j,  rho = 1 - sum_j w_j,  v_t(p) = rho d_0(p) + sum_j w_j d_t(p + o_j),
 *   d_{t+1} = m s + (1 - m) v_t  (d_{t+1} = v_t without samples)
 * and out = d_N.  Order of operations (DESIGN.md section 4.23): w is one rounded product; the sum adds j ascending from w_0;
 * v starts from the rounded product rho d_0 and adds the taps j = K*K-1 down to 0 by FMA, the centre included.
 * The backward writes any of grad_affinity [B][K*K][H][W], grad_attention [B][iters*(R+1)][H][W], grad_blur [B][C][H][W],
 * grad_sparse and grad_confidence [B][1][H][W] that is not NULL (the last two need the samples) and skips the work only the
 * NULL ones need: without grad_affinity, grad_attention and grad_confidence it recomputes no iterate.  iters = 0: attention
 * and grad_attention may be NULL (they have no channels); the forward copies blur to out, the backward copies grad_out and
 * zero-fills grad_affinity, grad_sparse and grad_confidence (cudaMemsetAsync).
 * Workspace (bytes, device-independent; the queries return 0 for invalid arguments): forward 4 * B*C*H*W for iters >= 2,
 * else 0; backward 4 * (2 * iters - 1) * B*C*H*W (lambda_0 .. lambda_{N-1} and d_1 .. d_{N-1}), 0 for iters = 0.
 * Launches: forward iters; backward at most (iters - 1) + iters + 1.  No atomics; the bits depend on the arguments only.
 * CSPN_ERR_INVALID_ARGUMENT for a null affinity / blur / out (grad_out in the backward), a null attention with iters > 0,
 * exactly one of sparse and confidence, a grad_sparse or grad_confidence without the samples, a non-positive shape, K not
 * in {3, 5, 7}, iters < 0, a pointer that is not 4-byte aligned, and an output (the workspace included) that overlaps an
 * input or another output; CSPN_ERR_UNSUPPORTED for B*C > 65535 or ceil(H/16) > 65535; CSPN_ERR_WORKSPACE for a missing or
 * short workspace.  All of these come before any device work. */
CSPN_API size_t cspn2d_dyn_workspace_bytes(int B, int C, int H, int W, int K, int iters);

CSPN_API int cspn2d_dyn_fwd_f32(const float* affinity, const float* attention, const float* blur, const float* sparse,
                       const float* confidence, float* out, int B, int C, int H, int W, int K, int iters, void* workspace,
                       size_t workspace_bytes, cspn_stream_t stream);

CSPN_API size_t cspn2d_dyn_bwd_workspace_bytes(int B, int C, int H, int W, int K, int iters);

CSPN_API int cspn2d_dyn_bwd_f32(const float* affinity, const float* attention, const float* blur, const float* sparse,
                       const float* confidence, const float* grad_out, float* grad_affinity, float* grad_attention,
                       float* grad_blur, float* grad_sparse, float* grad_confidence, int B, int C, int H, int W, int K,
                       int iters, void* workspace, size_t workspace_bytes, cspn_stream_t stream);

/* ---- 2D linear three-way scans: SPN's propagation (Liu et al., NIPS 2017; DESIGN.md section 4.24) -------------------
 * feat [B][C][H][W] is scanned in every direction of dir_mask (bit 0 l2r, 1 r2l, 2 t2b, 3 b2t; nd set bits, 1 .. 4,
 * taken in that canonical order).  For l2r (scan index t the column, lateral index i the row), with g_j = gate_j[i][t]
 * used as given (no abs, no normalisation) and reads outside the image 0:
 *   c = ((1 - g0) - g1) - g2,   h[i][t] = fma(g2, h[i+1][t-1], fma(g1, h[i][t-1], fma(g0, h[i-1][t-1], c * x[i][t])))
 * r2l reads column t + 1; t2b and b2t scan rows and read row y -+ 1 at columns x - 1, x, x + 1: tap j is lateral offset
 * j - 1 along increasing index in every direction.  gate_mode CSPN_LIN_GATE_SHARED: gate [B][3*nd][H][W], shared by the
 * C channels; CSPN_LIN_GATE_PER_CHANNEL: gate [B][3*nd*C][H][W].  Direction block k (the k-th requested direction) is
 * channels [3k*Cg, 3(k+1)*Cg), Cg = 1 or C, and channel c uses 3c .. 3c+2 within it.  out [B][C][H][W] is h for one
 * direction, else the node-wise max: h of the first direction that is NaN there, else of the first attaining the maximum.
 * planes [nd][B][C][H][W] (optional, nd > 1 only; NULL for nd = 1) receives every direction's h; without it the planes go
 * to the workspace.  The backward takes the planes (for nd = 1 the forward's out), routes grad_out to the direction the
 * merge picked, runs the adjoint scans in reverse and writes grad_feat [B][C][H][W] and grad_gate (laid out as gate),
 * whichever is not NULL: grad_feat sums the directions in canonical order, a shared gate's gradient sums the channels
 * c ascending (DESIGN.md section 4.24 gives every operation's order).
 * Workspace (bytes, device-independent; the queries return 0 for invalid arguments): forward 4 * nd * B*C*H*W for
 * nd > 1 (0 when planes is given), else 0; backward, for nd > 1, 8 * nd * B*C*H*W (grad_feat's per-direction planes
 * and the routed grad_out), and, for a shared gate with C > 1, 12 * nd * B*C*H*W.  Launches: forward 1 (nd = 1) or 2; backward at most 3.  No
 * atomics and no memsets; the bits depend on the arguments only.
 * CSPN_ERR_INVALID_ARGUMENT for a null feat / gate / out (planes / grad_out in the backward), planes given with nd = 1,
 * dir_mask outside 1 .. 15, an unknown gate_mode, a non-positive shape, a pointer that is not 4-byte aligned, and an
 * output (the workspace included) that overlaps an input or another output; CSPN_ERR_UNSUPPORTED for B*C times the
 * cluster size (1 .. 8, chosen from the shape) past 2^31 - 1 or a lateral extent (H for l2r / r2l, W for t2b / b2t) past 2048; CSPN_ERR_WORKSPACE for a missing or short workspace.  All
 * of these come before any device work. */
#define CSPN_LIN_GATE_SHARED 0
#define CSPN_LIN_GATE_PER_CHANNEL 1

CSPN_API size_t cspn2d_lin_workspace_bytes(int B, int C, int H, int W, int dir_mask, int gate_mode);

CSPN_API int cspn2d_lin_fwd_f32(const float* feat, const float* gate, float* out, float* planes, int B, int C, int H, int W,
                       int dir_mask, int gate_mode, void* workspace, size_t workspace_bytes, cspn_stream_t stream);

CSPN_API size_t cspn2d_lin_bwd_workspace_bytes(int B, int C, int H, int W, int dir_mask, int gate_mode);

CSPN_API int cspn2d_lin_bwd_f32(const float* feat, const float* gate, const float* planes, const float* grad_out,
                       float* grad_feat, float* grad_gate, int B, int C, int H, int W, int dir_mask, int gate_mode,
                       void* workspace, size_t workspace_bytes, cspn_stream_t stream);

/* ---- 2D with the Paddle module's own-location gates, K in {3, 5, 7} (CSPN.cspn with dimNum = 2, demo.py:20-54) -----
 * w_k(p) = |g_k(p)| / sum_j |g_j(p)| at the pixel's own location (IEEE division: a zero sum gives NaN), then iters steps
 * d_{t+1}(p) = sum_k w_k(p) d_t(p + off_k) with zero padding, no centre term and no sparse replacement.  Taps as in the
 * K x K calls above.  guidance [B][K*K-1][H][W], one gate shared by the C channels of feat [B][C][H][W]; per-channel gates
 * (demo.py:28-45, guidance [B][(K*K-1)*C][H][W]) are the same memory as B*C images with C = 1.  out / grad_feat
 * [B][C][H][W], grad_guidance [B][K*K-1][H][W]; either gradient may be NULL.  K = 3 runs on the K x K kernels too.
 * Workspace: forward B*K*K*H*W + B*C*H*W floats, backward B*K*K*H*W + 2*iters*B*C*H*W floats, 0 for iters == 0; neither
 * depends on the device.  CSPN_ERR_INVALID_ARGUMENT for K not in {3, 5, 7}, iters < 0, a non-positive shape or a null
 * guidance / feat / out (grad_out in the backward); CSPN_ERR_UNSUPPORTED for B*C > 65535. */
CSPN_API size_t cspn2d_paddle_workspace_bytes(int B, int C, int H, int W, int K, int iters);

CSPN_API int cspn2d_paddle_fwd_f32(const float* guidance, const float* feat, float* out,
                          int B, int C, int H, int W, int K, int iters,
                          void* workspace, size_t workspace_bytes, cspn_stream_t stream);

/* cspn2d_paddle_fwd_f32 fused with the final gather of a data-parallel run: see cspn2d_k_fwd_gather_f32 */
CSPN_API int cspn2d_paddle_fwd_gather_f32(const float* guidance, const float* feat, float* out,
                                 float* const* peer_out, int n_peer, float* multicast_out,
                                 int B, int C, int H, int W, int K, int iters,
                                 void* workspace, size_t workspace_bytes, cspn_stream_t stream);

CSPN_API size_t cspn2d_paddle_bwd_workspace_bytes(int B, int C, int H, int W, int K, int iters);

CSPN_API int cspn2d_paddle_bwd_f32(const float* guidance, const float* feat, const float* grad_out,
                          float* grad_guidance, float* grad_feat, int B, int C, int H, int W, int K, int iters,
                          void* workspace, size_t workspace_bytes, cspn_stream_t stream);

/* ---- 3D: replaces CSPN.cspn(guide, feat) (cspn_paddle/demo.py:20-54) ------------------------
 * guidance [B][26][D][H][W], feat/out [B][C][D][H][W] (gate shared across C, cspn_paddle/README.md:56)
 */
CSPN_API size_t cspn3d_workspace_bytes(int B, int C, int D, int H, int W, int iters);

CSPN_API int cspn3d_fwd_f32(const float* guidance, const float* feat, float* out,
                   int B, int C, int D, int H, int W, int iters, int norm_type,
                   void* workspace, size_t workspace_bytes, cspn_stream_t stream);

/* ---- fused gather of the 3D forwards -------------------------------------------------------------------------------
 * cspn3d_fwd_gather_f32, cspn3d_k_fwd_gather_f32 and cspn3d_gates_fwd_gather_f32 take the arguments of their plain forward
 * plus peer_out / n_peer / multicast_out after `out`, exactly as the 2D gathers do (see cspn2d_k_fwd_gather_f32), and give
 * `out` its bits.  The last step of the forward also stores its result to each peer_out[i] (the same [B][C][D][H][W]
 * block inside another GPU's gather buffer) and / or to multicast_out; intermediate steps stay local.  Same checks and
 * codes as in 2D: n_peer 0..7 with a non-null array when non-zero, every peer_out[i] non-null, every peer_out[i] and
 * multicast_out (may be NULL) 16-byte aligned, else CSPN_ERR_INVALID_ARGUMENT; iters == 0 is CSPN_ERR_UNSUPPORTED.
 * Workspace as for the plain forward (its *_workspace_bytes), and cspn_last_launches() counts the same launches.
 * K = 3 in cspn3d_k_fwd_gather_f32 delegates to cspn3d_fwd_gather_f32; every entry takes any W.  Per-channel gates are
 * B*C volumes with C = 1, as in the plain calls: the output memory, and with it the peer offsets, is the same.  The
 * caller orders the remote stores before their consumers (a barrier across ranks after the call). */
CSPN_API int cspn3d_fwd_gather_f32(const float* guidance, const float* feat, float* out,
                          float* const* peer_out, int n_peer, float* multicast_out,
                          int B, int C, int D, int H, int W, int iters, int norm_type,
                          void* workspace, size_t workspace_bytes, cspn_stream_t stream);

CSPN_API int cspn3d_fwd_f32_host(const float* guidance, const float* feat, float* out,
                        int B, int C, int D, int H, int W, int iters, int norm_type, int device);

/* ---- 3D backward (the Paddle op trains too: cspn_paddle/demo.py:72-75 minimises a loss through it).
 * grad_guidance [B][26][D][H][W], grad_feat [B][C][D][H][W]; either may be NULL.  Workspace (27 + (2*iters-1)*C)*D*H*W
 * floats, 0 for iters == 0 (one volume at a time; independent of B and of the device). */
CSPN_API size_t cspn3d_bwd_workspace_bytes(int B, int C, int D, int H, int W, int iters);

CSPN_API int cspn3d_bwd_f32(const float* guidance, const float* feat, const float* grad_out,
                   float* grad_guidance, float* grad_feat,
                   int B, int C, int D, int H, int W, int iters, int norm_type,
                   void* workspace, size_t workspace_bytes, cspn_stream_t stream);

/* ---- 3D with a K x K x K affinity kernel, K in {3, 5} (K^3-1 = 26, 124 neighbours) ---------------------------------
 * Tap k enumerates (f, t, l) over [0,K)^3 in raster order without the centre and reads the source at
 * (dz, dy, dx) = ((K-1)/2 - f, (K-1)/2 - t, (K-1)/2 - l) (DESIGN.md section 4.9).
 * guidance [B][K^3-1][D][H][W] (one gate shared by the C channels of feat), feat / out / grad_* [B][C][D][H][W];
 * norm_type is a cspn_norm3d (0 gathered signed, 1 gathered abs, 2 own-location 'paddle').
 * K = 3 is the 3D operator above: cspn3d_fwd_f32 / cspn3d_bwd_f32 are these calls at K = 3, with the same results and
 * workspace queries.  Forward workspace G*(K^3 + (iters > 1 ? C : 0))*D*H*W floats, with G the volumes per launch group
 * (all B unless that exceeds 4 GiB or gridDim.z); backward (K^3 + (2*iters-1)*C)*D*H*W floats; 0 for iters == 0; neither
 * depends on the device.  CSPN_ERR_INVALID_ARGUMENT for K not in {3, 5}, an unknown norm, iters < 0, a non-positive shape or a null
 * guidance / feat / out (grad_out in the backward; grad_guidance and grad_feat may be NULL).  CSPN_ERR_UNSUPPORTED for a
 * shape the launch grid cannot take (D*C > 65535). */
CSPN_API size_t cspn3d_k_workspace_bytes(int B, int C, int D, int H, int W, int K, int iters);

CSPN_API int cspn3d_k_fwd_f32(const float* guidance, const float* feat, float* out,
                     int B, int C, int D, int H, int W, int K, int iters, int norm_type,
                     void* workspace, size_t workspace_bytes, cspn_stream_t stream);

/* cspn3d_k_fwd_f32 fused with the final gather of a data-parallel run: see cspn3d_fwd_gather_f32 */
CSPN_API int cspn3d_k_fwd_gather_f32(const float* guidance, const float* feat, float* out,
                            float* const* peer_out, int n_peer, float* multicast_out,
                            int B, int C, int D, int H, int W, int K, int iters, int norm_type,
                            void* workspace, size_t workspace_bytes, cspn_stream_t stream);

CSPN_API size_t cspn3d_k_bwd_workspace_bytes(int B, int C, int D, int H, int W, int K, int iters);

CSPN_API int cspn3d_k_bwd_f32(const float* guidance, const float* feat, const float* grad_out,
                     float* grad_guidance, float* grad_feat,
                     int B, int C, int D, int H, int W, int K, int iters, int norm_type,
                     void* workspace, size_t workspace_bytes, cspn_stream_t stream);

/* ---- caller-supplied gates: fluid.layers.affinity_propagate(input, gate_weight, kernel_size) itself -----------------
 * The Paddle op the reference calls once per step (cspn_paddle/demo.py:41-43, 51-52), with its gates already normalised by
 * the caller (cspn_paddle/README.md:54), run `iters` times:
 *   d_{t+1}(p) = sum_k g_k(p) d_t(p + off_k),  d_0 = feat,
 * with the gates used exactly as given (no |.|, no normalisation, no centre term, no sparse replacement), zero padding and
 * IEEE arithmetic (inf * 0 = NaN where a tap reads the padding).  Taps as in the K x K (2D) and K x K x K (3D) calls above.
 * gates [B][K^d-1][(D)][H][W], one gate shared by the C channels of feat / out / grad_feat [B][C][(D)][H][W]; per-channel
 * gates (demo.py:28-45, [B][(K^d-1)*C]...) are the same memory as B*C volumes with C = 1.  grad_gates has the shape of
 * gates; either gradient may be NULL, and the backward then skips the work that only feeds it (without grad_gates it
 * runs the adjoint steps alone).  2D: K in {3, 5, 7}; 3D: K in {3, 5}.
 * Workspace (0 for iters == 0; none depends on the device):
 *   2D forward   B*C*H*W floats for iters >= 2, else 0;
 *   2D backward  (2*iters-2)*B*C*H*W floats (lambda_0 is written straight into grad_feat);
 *   3D forward   G*C*D*H*W floats for iters >= 2, else 0, with G the volumes per launch group (all B unless that exceeds
 *                4 GiB or gridDim.z);
 *   3D backward  (2*iters-2)*C*D*H*W floats (one volume at a time; lambda_0 is written straight into grad_feat).
 * CSPN_ERR_INVALID_ARGUMENT for a bad K, iters < 0, a non-positive shape or a null gates / feat / out (grad_out in the
 * backward); CSPN_ERR_UNSUPPORTED for a shape the launch grid cannot take (B*C > 65535 in 2D, D*C > 65535 in 3D, or
 * H > 524280). */
CSPN_API size_t cspn2d_gates_workspace_bytes(int B, int C, int H, int W, int K, int iters);

CSPN_API int cspn2d_gates_fwd_f32(const float* gates, const float* feat, float* out,
                         int B, int C, int H, int W, int K, int iters,
                         void* workspace, size_t workspace_bytes, cspn_stream_t stream);

/* cspn2d_gates_fwd_f32 fused with the final gather of a data-parallel run: see cspn2d_k_fwd_gather_f32 */
CSPN_API int cspn2d_gates_fwd_gather_f32(const float* gates, const float* feat, float* out,
                                float* const* peer_out, int n_peer, float* multicast_out,
                                int B, int C, int H, int W, int K, int iters,
                                void* workspace, size_t workspace_bytes, cspn_stream_t stream);

CSPN_API size_t cspn2d_gates_bwd_workspace_bytes(int B, int C, int H, int W, int K, int iters);

CSPN_API int cspn2d_gates_bwd_f32(const float* gates, const float* feat, const float* grad_out,
                         float* grad_gates, float* grad_feat, int B, int C, int H, int W, int K, int iters,
                         void* workspace, size_t workspace_bytes, cspn_stream_t stream);

CSPN_API size_t cspn3d_gates_workspace_bytes(int B, int C, int D, int H, int W, int K, int iters);

CSPN_API int cspn3d_gates_fwd_f32(const float* gates, const float* feat, float* out,
                         int B, int C, int D, int H, int W, int K, int iters,
                         void* workspace, size_t workspace_bytes, cspn_stream_t stream);

/* cspn3d_gates_fwd_f32 fused with the final gather of a data-parallel run: see cspn3d_fwd_gather_f32 */
CSPN_API int cspn3d_gates_fwd_gather_f32(const float* gates, const float* feat, float* out,
                                float* const* peer_out, int n_peer, float* multicast_out,
                                int B, int C, int D, int H, int W, int K, int iters,
                                void* workspace, size_t workspace_bytes, cspn_stream_t stream);

CSPN_API size_t cspn3d_gates_bwd_workspace_bytes(int B, int C, int D, int H, int W, int K, int iters);

CSPN_API int cspn3d_gates_bwd_f32(const float* gates, const float* feat, const float* grad_out,
                         float* grad_gates, float* grad_feat, int B, int C, int D, int H, int W, int K, int iters,
                         void* workspace, size_t workspace_bytes, cspn_stream_t stream);

/* ---- the guidance and depth heads: Unpool + crop + 3x3 convolution in one kernel -----------------------------------
 * Simple_Gudi_UpConv_Block_Last_Layer (torch_resnet_cspn_nyu.py:187-205): u = Unpool(x) (conv_transpose2d with a [1,0;0,0]
 * kernel, stride 2, groups=Cin: u(2i, 2j) = x(i, j), the other three cells of each 2x2 block x(i, j) * 0), cropped to
 * H x W, then out = conv2d(u, weight, padding=1, no bias):
 *   out(co, p) = sum_ci sum_tap weight[co][ci][ky][kx] * u(ci, p + (ky-1, kx-1)),  zero padding.
 * x [B][Cin][h][w], weight [Cout][Cin][3][3], out / grad_out [B][Cout][H][W] with 1 <= H <= 2h, 1 <= W <= 2w; grad_x has
 * the shape of x and grad_weight that of weight.  Any Cin, Cout >= 1; every pointer 4-byte aligned.
 * IEEE as the op sequence: the products with the structural zeros (inserted cells, padding) are skipped, and the forward
 * puts back the NaN they give for a non-finite x or weight.  The backward is exact for finite inputs only: gradients flow
 * through the real cells, so a non-finite value is not spread by a product with a structural zero.
 * Every sum has a fixed order: the forward and grad_x bits of an image do not depend on the rest of the batch, and
 * grad_weight is the same from run to run (per-CTA partials in the workspace, summed in order by a second kernel).
 * The forward launches one kernel and needs no workspace.  The backward launches one kernel for grad_x and two for
 * grad_weight; either gradient may be NULL and its kernels are then skipped.  The workspace (4-byte aligned) is needed only
 * with grad_weight, cspn_unpool_conv3x3_bwd_workspace_bytes() bytes, which depends on the shape alone (0 for an invalid one).
 * No allocation, no synchronisation; cspn_last_launches() reports the kernels launched.
 * CSPN_ERR_INVALID_ARGUMENT for a non-positive size, H > 2h or W > 2w, a null x / weight / out (grad_out in the backward)
 * or a misaligned pointer; CSPN_ERR_WORKSPACE for a missing or short workspace; CSPN_ERR_UNSUPPORTED for a shape the launch
 * grid cannot take (B > 65535). */
CSPN_API int cspn_unpool_conv3x3_fwd_f32(const float* x, const float* weight, float* out, int B, int Cin, int h, int w,
                                int Cout, int H, int W, cspn_stream_t stream);

CSPN_API size_t cspn_unpool_conv3x3_bwd_workspace_bytes(int B, int Cin, int h, int w, int Cout, int H, int W);

CSPN_API int cspn_unpool_conv3x3_bwd_f32(const float* x, const float* weight, const float* grad_out, float* grad_x,
                                float* grad_weight, int B, int Cin, int h, int w, int Cout, int H, int W,
                                void* workspace, size_t workspace_bytes, cspn_stream_t stream);

/* ---- trilinear resampling: the Paddle module's resize_trilinear ---------------------------------------------------
 * fluid.layers.resize_trilinear (one of the Paddle wheel's two custom ops, cspn_paddle/README.md:24): x [B][C][D][H][W] -> out
 * [B][C][Do][Ho][Wo].  Per axis n_in -> n_out, in fp32, every operation rounded on its own:
 *   r = (n_in-1)/(n_out-1) if align_corners, else n_in/n_out; r = 0 when n_out == 1
 *   s(o) = max(r*(o+0.5) - 0.5, 0) if !align_corners && align_mode == 0, else r*o
 *   i0 = (int)s, i1 = i0 + (i0 < n_in-1), l1 = s - i0, l0 = 1 - l1
 *   out = l0d*(l0h*(l0w*x[d0,h0,w0] + l1w*x[d0,h0,w1]) + l1h*(...h1...)) + l1d*(...d1...), every product computed.
 * The backward is a gather (no atomics): grad_x[d,h,w] = sum_od (sum_oh (sum_ow g*ww) * wh) * wd over the outputs that read
 * the voxel, each sum from 0 in ascending o; the weight of (o, i) is l0 if i0(o) == i, else l1, and where i1 == i0 == i
 * both products are added (l0 first).  The bits depend on the arguments only (DESIGN.md section 4.14).
 * align_corners and align_mode are 0 or 1 (align_mode matters only without align_corners).  Every pointer 4-byte aligned;
 * out / grad_x must not overlap x / grad_out, nor the workspace either of them.  The forward launches one kernel and needs no workspace; the backward
 * launches two and writes every grad_x element.  Its workspace, cspn_resize_trilinear_bwd_workspace_bytes() bytes,
 * 8-byte aligned, depends on the six sizes alone (0 for a non-positive one).  No allocation, no synchronisation.
 * CSPN_ERR_INVALID_ARGUMENT for a null pointer, a non-positive size, an align flag outside {0, 1}, a misaligned or an
 * overlapping pointer (a workspace overlapping grad_x or grad_out included); CSPN_ERR_WORKSPACE for a missing, short or misaligned workspace; CSPN_ERR_UNSUPPORTED for an input
 * or output with >= 2^31 elements per (B*C) slice.  Any B*C is taken. */
CSPN_API int cspn_resize_trilinear_fwd_f32(const float* x, float* out, int B, int C, int D, int H, int W, int Do, int Ho,
                                  int Wo, int align_corners, int align_mode, cspn_stream_t stream);

CSPN_API size_t cspn_resize_trilinear_bwd_workspace_bytes(int D, int H, int W, int Do, int Ho, int Wo);

CSPN_API int cspn_resize_trilinear_bwd_f32(const float* grad_out, float* grad_x, int B, int C, int D, int H, int W, int Do,
                                  int Ho, int Wo, int align_corners, int align_mode, void* workspace,
                                  size_t workspace_bytes, cspn_stream_t stream);

/* ---- disparity regression from a low-resolution cost volume ---------------------------------------------------------
 * The soft-argmin head of GC-Net / PSMNet-style stereo networks on a cost volume cost [B][C][D][H][W], in one op:
 *   U = resize_trilinear(cost, (Do, Ho, Wo), align_corners, align_mode)     (the bits of cspn_resize_trilinear_fwd_f32)
 *   out[b][c][h][w] = sum_{o=0}^{Do-1} o * softmax_o(U[b][c][:][h][w])      out is [B][C][Ho][Wo]
 * The softmax subtracts the column maximum, uses expf, and sums S = sum e and N = sum o*e in ascending o; out = N / S.  A NaN
 * or +inf in the upsampled column, or a column all -inf, gives NaN.  The upsampled volume is never stored.
 * The backward recomputes the softmax from cost: gU_o = ((e_o * (g / S)) * (o - out)), then resize's adjoint as a gather
 * (along d per pixel, then sum_oh (sum_ow gv * w_w) * w_h per voxel, ascending, zero-weight taps included): no atomics,
 * every grad_cost element written once, the bits depend on the arguments only (DESIGN.md section 4.15).
 * Arguments and errors are cspn_resize_trilinear_*'s: align flags 0 or 1, every pointer 4-byte aligned, out / grad_cost
 * must not overlap cost (nor grad_out), and the workspace, cspn_disparity_regression_bwd_workspace_bytes() bytes (resize's
 * tables, 8*(Do+Ho+Wo+D+H+W)), 8-byte aligned, must overlap none of the three.  The forward launches one kernel, the
 * backward two.  No allocation, no synchronisation.  CSPN_ERR_UNSUPPORTED also for Do > 2^24 and for a shape whose 1x1 tile
 * of cost columns does not fit in shared memory: with Do = D, D above about 2150 without upsampling in H and W, above about
 * 520 at 4x (about 370 with align_corners = 0, align_mode = 0). */
CSPN_API int cspn_disparity_regression_fwd_f32(const float* cost, float* out, int B, int C, int D, int H, int W, int Do,
                                  int Ho, int Wo, int align_corners, int align_mode, cspn_stream_t stream);

CSPN_API size_t cspn_disparity_regression_bwd_workspace_bytes(int D, int H, int W, int Do, int Ho, int Wo);

CSPN_API int cspn_disparity_regression_bwd_f32(const float* cost, const float* grad_out, float* grad_cost, int B, int C,
                                  int D, int H, int W, int Do, int Ho, int Wo, int align_corners, int align_mode,
                                  void* workspace, size_t workspace_bytes, cspn_stream_t stream);

/* ---- stereo cost volumes from left and right feature maps ----------------------------------------------------------
 * left and right are [B][F][H][W] (the reference and the target image's features); D >= 1 disparities, the matched pixel
 * of left[..., x] at disparity d is right[..., x - d].  Cells with x < d are +0.0 whatever the inputs hold; D > W is allowed.
 *   concat (PSMNet):  out [B][2F][D][H][W]: out[b][c][d][y][x] = left[b][c][y][x], out[b][F+c][d][y][x] = right[b][c][y][x-d]
 *                     (copies: every bit is kept)
 *   gwc (GwcNet):     out [B][G][D][H][W], n = F / G: out[b][g][d][y][x] = (sum_{c in group g} left*right) / n, the products
 *                     summed in ascending c from the first, every operation rounded on its own
 * Backward, from grad_out (the volume's shape), both gradients [B][F][H][W], sums in ascending d from d = 0:
 *   concat:  grad_left[c][y][x] = sum_{d<=min(x,D-1)} g[c][d][y][x], grad_right[c][y][x] = sum_{d<=min(W-1-x,D-1)} g[F+c][d][y][x+d]
 *   gwc:     t = g / n;  grad_left = sum_d t[grp][d][y][x] * right[c][y][x-d],  grad_right = sum_d t[grp][d][y][x+d] * left[c][y][x+d]
 * No atomics, no workspace, every output element written once; the bits depend on the arguments only (DESIGN.md section
 * 4.16).  left may be right.  CSPN_ERR_INVALID_ARGUMENT for a null or not 4-byte aligned pointer, a size < 1, F % G != 0,
 * or an output that overlaps an input or the other output.  CSPN_ERR_UNSUPPORTED for 2F >= 2^31, D*H*W >= 2^31, and a D
 * whose 1-column tile does not fit in shared memory (concat: min(D, W) above about 14500; gwc: n * min(D, W) above about
 * 58000, or D above about 3200).  One launch each.  No allocation, no synchronisation. */
CSPN_API int cspn_concat_volume_fwd_f32(const float* left, const float* right, float* out, int B, int F, int H, int W, int D,
                                  cspn_stream_t stream);

CSPN_API int cspn_concat_volume_bwd_f32(const float* grad_out, float* grad_left, float* grad_right, int B, int F, int H,
                                  int W, int D, cspn_stream_t stream);

CSPN_API int cspn_gwc_volume_fwd_f32(const float* left, const float* right, float* out, int B, int F, int H, int W, int D,
                                  int G, cspn_stream_t stream);

CSPN_API int cspn_gwc_volume_bwd_f32(const float* left, const float* right, const float* grad_out, float* grad_left,
                                  float* grad_right, int B, int F, int H, int W, int D, int G, cspn_stream_t stream);

/* ---- affinity pooling: the CSPN stereo network's convolutional spatial pyramid pooling --------------------------------
 * feat [B][C][H][W]; gate [B][L][H][W], channel l the raw affinity of level l, shared by all C channels; kernel_sizes a HOST
 * array of L ints, 1 <= L <= 8, each 1 <= p_l <= min(H, W), in any order, repeats allowed.  Level l pools the windows of
 * avg_pool2d(x, p_l) (stride p_l, no padding, floor mode) into [B][C][H/p_l][W/p_l]:
 *   a = |gate_l|,  S = sum_window a,  w = a / S,  out_l[b][c][i][j] = sum_window w * feat[b][c]
 * out and grad_out are one buffer, level-major: level l starts at B*C*sum_{l'<l} (H/p_l')*(W/p_l').  The order: each window
 * row summed in ascending x, then the row sums in ascending y (S and out alike); backward
 *   grad_feat[c][q] = sum over the levels that cover q, ascending l, of w_l(q) * grad_out_l[c][cell], +0.0 if none covers q
 *   grad_gate_l[q]  = ((sum_c grad_out_l[c][cell] * (feat[c][q] - out_l[c][cell]), ascending c) / S) * sgn(gate_l[q]),
 *                     +0.0 outside level l's windows
 * every operation rounded on its own, every sum from its first term (DESIGN.md section 4.17).  An all-zero window gives
 * NaN (0/0) in every channel of its cell.  No atomics, no workspace, every output element written once; the bits depend on
 * the arguments only.  CSPN_ERR_INVALID_ARGUMENT for a null or not 4-byte aligned pointer, a size < 1, L outside [1, 8],
 * a null kernel_sizes or a p_l outside [1, min(H, W)], and an output that overlaps an input or the other output.
 * CSPN_ERR_UNSUPPORTED for H*W >= 2^31 and a grid past 2^31 - 1 blocks.  One launch each.  No allocation, no
 * synchronisation. */
CSPN_API int cspn_affinity_pool2d_fwd_f32(const float* feat, const float* gate, float* out, int B, int C, int H, int W,
                                  int L, const int* kernel_sizes, cspn_stream_t stream);

CSPN_API int cspn_affinity_pool2d_bwd_f32(const float* feat, const float* gate, const float* out, const float* grad_out,
                                  float* grad_feat, float* grad_gate, int B, int C, int H, int W, int L,
                                  const int* kernel_sizes, cspn_stream_t stream);

/* ---- affinity fusion: the CSPN stereo network's spatial pyramid fusion --------------------------------------------------
 * levels a HOST array of L DEVICE pointers, level l [B][C][h_l][w_l]; level_hw a HOST array (h_0, w_0, h_1, w_1, ...) of 2L
 * ints, 1 <= L <= 8, any h_l, w_l >= 1 (a level may be finer than the output); gate [B][L][H][W], channel l the raw
 * affinity of level l, shared by all C channels; out [B][C][H][W].  At every pixel q:
 *   a_l = |gate_l(q)|,  S = sum_l a_l,  w_l = a_l / S,  out[c](q) = sum_l w_l * u_l[c](q)
 * u_l is level l resampled bilinearly to H x W with resize_trilinear's per-axis rule (align_corners, align_mode as there):
 *   u = l0h*(l0w*x[h0][w0] + l1w*x[h0][w1]) + l1h*(l0w*x[h1][w0] + l1w*x[h1][w1]), every product computed.
 * S and out summed in ascending l from the first term; backward
 *   grad_gate_l(q) = ((sum_c grad_out[c](q) * (u_l[c](q) - out[c](q)), ascending c) / S) * sgn(gate_l(q))
 *   grad_levels[l] = resize_trilinear's gather over H and W of v = w_l * grad_out: sum_oh (sum_ow v * lw) * lh, each sum
 *                    from 0 in ascending o, both products (v * l0 first) where i1 == i0; +0.0 where no output reads a cell
 * every operation rounded on its own (DESIGN.md section 4.18).  All-zero gates at a pixel give NaN (0/0) in every channel
 * there.  Levels may alias one another (the caller adds their gradients).  CSPN_ERR_INVALID_ARGUMENT for a null or not
 * 4-byte aligned pointer, a size < 1, L outside [1, 8], an align flag outside {0, 1}, and an output (the workspace
 * included) that overlaps an input or another output.  CSPN_ERR_UNSUPPORTED for H*W >= 2^31 or h_l*w_l >= 2^31 (the grids
 * then stay within their limits).  No atomics, no memset, every output element written once; the bits depend on the
 * arguments only.  The forward is one launch; the backward three, with
 * cspn_affinity_fuse2d_bwd_workspace_bytes() bytes of 4-byte aligned workspace (0 for invalid sizes).  No allocation, no
 * synchronisation. */
CSPN_API int cspn_affinity_fuse2d_fwd_f32(const float* const* levels, const int* level_hw, const float* gate, float* out,
                                  int B, int C, int H, int W, int L, int align_corners, int align_mode,
                                  cspn_stream_t stream);

CSPN_API size_t cspn_affinity_fuse2d_bwd_workspace_bytes(int B, int C, int H, int W, int L, const int* level_hw);

CSPN_API int cspn_affinity_fuse2d_bwd_f32(const float* const* levels, const int* level_hw, const float* gate,
                                  const float* out, const float* grad_out, float* const* grad_levels, float* grad_gate,
                                  int B, int C, int H, int W, int L, int align_corners, int align_mode, void* workspace,
                                  size_t workspace_bytes, cspn_stream_t stream);

/* ---- atrous affinity pooling: the CSPN stereo network's atrous spatial pyramid pooling (ACSPP) --------------------------
 * feat [B][C][H][W]; dilations a HOST array of L ints, 1 <= L <= 8, each 1 <= r_l <= max(H, W), in any order, repeats
 * allowed; gate [B][9L][H][W], channel 9l + t the raw affinity of tap t of level l, offset (dy, dx) = (t/3 - 1, t%3 - 1)
 * (tap 4 the centre, learned like the others), shared by all C channels; out [B][L*C][H][W], channels lC .. lC + C - 1
 * level l.  At every pixel p, with r = r_l and feat = +0.0 outside the image (a tap there still counts in S):
 *   a_t = |gate[9l + t](p)|,  S = sum_t a_t,  w_t = a_t / S,  out[lC + c](p) = sum_t w_t * feat[c](p + r (dy_t, dx_t))
 * S and out summed in ascending t from the first term; backward
 *   grad_gate[9l + t](p) = ((sum_c grad_out[lC + c](p) * (feat[c](p + r d_t) - out[lC + c](p)), ascending c) / S) * sgn(gate)
 *   grad_feat[c](q)      = sum over l ascending, then t ascending, of w_{l,t}(q - r_l d_t) * grad_out[lC + c](q - r_l d_t),
 *                          over the terms whose source pixel lies in the image
 * every operation rounded on its own (DESIGN.md section 4.19).  All-zero gates of a level at a pixel give NaN (0/0) in
 * every channel of that level there.  CSPN_ERR_INVALID_ARGUMENT for a null or not 4-byte aligned pointer, a size < 1,
 * L outside [1, 8], a null dilations or an r_l outside [1, max(H, W)], and an output (the workspace included) that
 * overlaps an input or another output; CSPN_ERR_WORKSPACE for a null, short or not 4-byte aligned workspace.
 * CSPN_ERR_UNSUPPORTED for H*W >= 2^31 and a grid of 2^31 blocks or more.  No atomics, no memset, every output element
 * written once; the bits depend on the arguments only.  The forward is one launch; the backward two, with
 * cspn_affinity_atrous2d_bwd_workspace_bytes() bytes of 4-byte aligned workspace (4 * B*9L*H*W, the weight planes; 0 for
 * invalid arguments).  No allocation, no synchronisation. */
CSPN_API int cspn_affinity_atrous2d_fwd_f32(const float* feat, const float* gate, float* out, int B, int C, int H, int W,
                                    int L, const int* dilations, cspn_stream_t stream);

CSPN_API size_t cspn_affinity_atrous2d_bwd_workspace_bytes(int B, int C, int H, int W, int L, const int* dilations);

CSPN_API int cspn_affinity_atrous2d_bwd_f32(const float* feat, const float* gate, const float* out, const float* grad_out,
                                    float* grad_feat, float* grad_gate, int B, int C, int H, int W, int L,
                                    const int* dilations, void* workspace, size_t workspace_bytes, cspn_stream_t stream);

/* ---- what the reference does with the result on the HOST after every step, on the device ------------------------
 * utils.evaluate_error(gt_depth, pred_depth) (cspn_pytorch/utils.py:19-47; called at train.py:206, eval.py:150 after a
 * `.cpu()` of both tensors) and Wighted_L1_Loss (loss.py:12-23).  One pass over n = B*C*H*W elements; out12 (DEVICE):
 *   [0] n_valid (gt > 1e-4)  [1] MSE  [2] RMSE  [3] MAE (== the masked L1 loss)  [4] ABS_REL
 *   [5..10] DELTA1.02, 1.05, 1.10, 1.25, 1.25^2, 1.25^3   [11] reserved (LG10: never filled by the reference)
 * workspace: cspn_depth_metrics_workspace_bytes() bytes of 8-byte aligned device memory.  Enqueue only, no sync. */
CSPN_API size_t cspn_depth_metrics_workspace_bytes(void);
CSPN_API int cspn_depth_metrics_f32(const float* pred, const float* gt, size_t n, float* out12,
                           void* workspace, size_t workspace_bytes, cspn_stream_t stream);
/* gradient of the masked L1 loss w.r.t. pred: grad_loss (device scalar, NULL = 1) * sign(pred - gt) / n_valid where
 * gt > 1e-4, else 0; stats12 is the out12 of cspn_depth_metrics_f32 on the same tensors (autograd through loss.py:16-23) */
CSPN_API int cspn_masked_l1_bwd_f32(const float* pred, const float* gt, const float* stats12, const float* grad_loss,
                           float* grad_pred, size_t n, cspn_stream_t stream);

/* ---- pinned host buffers for the *_host entry points ---------------------------------------- */
CSPN_API void* cspn_host_alloc(size_t bytes); /* cudaHostAlloc; NULL on failure */
CSPN_API void cspn_host_free(void* p);

/* ---- introspection --------------------------------------------------------------------------- */
CSPN_API const char* cspn_last_error(void);   /* thread-local, never NULL */
CSPN_API int cspn_version(void);              /* 10000*major + 100*minor + patch */
CSPN_API int cspn_last_algo(void);            /* cspn_algo actually used by this thread's last 2D forward */
CSPN_API int cspn_last_launches(void);        /* kernels this thread's last call launched */
/* Human-readable plan for a 2D shape (tile geometry, cluster size, strips); returns bytes written. */
CSPN_API int cspn2d_describe_plan(int B, int C, int H, int W, int iters, int algo, char* buf, int buf_len);
/* The cluster path's plan as JSON: passes (count, steps, tile geometry) with their strips [tile_x0, ux0, ux1] and
 * row bands [band_y0, uy0, uy1]; {"supported": false, ...} when the shape goes to the generic path.  Returns the
 * bytes needed (output is truncated to buf_len). */
CSPN_API int cspn2d_plan_json(int H, int W, int iters, char* buf, int buf_len);
/* The same for the CHAINED plan: the strips of an image are processed left to right and every strip hands the column left
 * of its right neighbour on, step by step, so only a strip's right edge goes stale (fewer, more useful strips).  The
 * forward uses it for large batches when the caller's workspace holds cspn2d_workspace_bytes(); "supported": false when
 * the shape has no such plan (one strip, row bands, more than 32 steps per pass). */
CSPN_API int cspn2d_plan_json_chained(int H, int W, int iters, char* buf, int buf_len);

#ifdef __cplusplus
}
#endif
#endif /* CSPN_B200_H_ */
