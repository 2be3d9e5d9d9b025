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
 * grad_blur [B][C][H][W].  Either may be NULL.  Needs the forward inputs again. */
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
 * queries return theirs.  K = 5 / 7: forward workspace B*K*K*H*W + B*C*H*W floats, backward B*K*K*H*W + 2*iters*B*C*H*W
 * floats (0 for iters == 0); the size does not depend on the device.  CSPN_ERR_INVALID_ARGUMENT for K not in {3, 5, 7},
 * guidance_channels < K*K-1, an unknown norm, iters < 0, a non-positive shape or a null guidance / blur / out
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
 * grad_guidance [B][26][D][H][W], grad_feat [B][C][D][H][W]; either may be NULL. */
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
 * K = 3 IS the 3D operator: the calls delegate to cspn3d_fwd_f32 / cspn3d_bwd_f32 and the workspace queries return theirs.
 * K = 5: forward workspace G*(125 + (iters > 1 ? C : 0))*D*H*W floats, with G the volumes per launch group (all B unless
 * that exceeds 4 GiB or gridDim.z); backward (125 + (2*iters-1)*C)*D*H*W floats; 0 for iters == 0; neither depends on the
 * device.  CSPN_ERR_INVALID_ARGUMENT for K not in {3, 5}, an unknown norm, iters < 0, a non-positive shape or a null
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
