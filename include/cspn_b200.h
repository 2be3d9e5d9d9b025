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
 * cspn2d_workspace_bytes(..., CSPN_ALGO_GENERIC) as the size to provide. */
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

/* ---- 3D: replaces CSPN.cspn(guide, feat) (cspn_paddle/demo.py:20-54) ------------------------
 * guidance [B][26][D][H][W], feat/out [B][C][D][H][W] (gate shared across C, cspn_paddle/README.md:56)
 */
CSPN_API size_t cspn3d_workspace_bytes(int B, int C, int D, int H, int W, int iters);

CSPN_API int cspn3d_fwd_f32(const float* guidance, const float* feat, float* out,
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
