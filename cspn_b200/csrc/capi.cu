// extern "C" surface of libcspn_b200.so (include/cspn_b200.h): argument checking, algorithm
// dispatch, and the chunked host-buffer pipeline behind the *_host entry points.
#include <cstdlib>
#include <mutex>
#include <vector>

#include "common.cuh"

namespace cspn {

static thread_local char g_err[512] = "";
thread_local int g_last_algo = 0;
thread_local int g_last_launches = 0;

void set_error(const char* fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
}
void clear_error() { g_err[0] = 0; }

namespace {

struct DeviceGuard {
    int prev = -1;
    bool ok = true;
    explicit DeviceGuard(int dev) {
        if (cudaGetDevice(&prev) != cudaSuccess) { ok = false; return; }
        if (dev >= 0 && dev != prev && cudaSetDevice(dev) != cudaSuccess) ok = false;
    }
    ~DeviceGuard() {
        if (prev >= 0) cudaSetDevice(prev);
    }
};

int device_of(const void* p) {
    cudaPointerAttributes a;
    if (cudaPointerGetAttributes(&a, p) != cudaSuccess) { cudaGetLastError(); return -1; }
    return (a.type == cudaMemoryTypeDevice || a.type == cudaMemoryTypeManaged) ? a.device : -1;
}

int check2d(const float* guidance, const float* blur, float* out, int B, int C, int H, int W, int gch, int iters,
            int norm_type, int algo) {
    if (!guidance || !blur || !out) { set_error("null tensor pointer"); return CSPN_ERR_INVALID_ARGUMENT; }
    if (B <= 0 || C <= 0 || H <= 0 || W <= 0) { set_error("non-positive shape B=%d C=%d H=%d W=%d", B, C, H, W); return CSPN_ERR_INVALID_ARGUMENT; }
    if (gch < 8) { set_error("guidance needs >= 8 channels, got %d (cspn.py:91-98)", gch); return CSPN_ERR_INVALID_ARGUMENT; }
    if (iters < 0) { set_error("prop_time must be >= 0, got %d", iters); return CSPN_ERR_INVALID_ARGUMENT; }
    if (norm_type != CSPN_NORM_8SUM && norm_type != CSPN_NORM_8SUM_ABS) { set_error("unknown norm_type %d (cspn.py:36)", norm_type); return CSPN_ERR_INVALID_ARGUMENT; }
    if (algo < CSPN_ALGO_AUTO || algo > CSPN_ALGO_CLUSTER) { set_error("unknown algo %d", algo); return CSPN_ERR_INVALID_ARGUMENT; }
    return CSPN_OK;
}

// The destinations of a fused gather (cspn{2,3}d_*fwd_gather_f32) and its step count: the checks every gather entry shares
int check_gather(float* const* peer_out, int n_peer, const float* multicast_out, int iters) {
    if (n_peer < 0 || n_peer > 7 || (n_peer > 0 && !peer_out)) { set_error("n_peer must be 0..7 with a pointer array"); return CSPN_ERR_INVALID_ARGUMENT; }
    for (int i = 0; i < n_peer; ++i)
        if (!peer_out[i] || (reinterpret_cast<uintptr_t>(peer_out[i]) & 15)) { set_error("peer_out[%d] is null or not 16-byte aligned", i); return CSPN_ERR_INVALID_ARGUMENT; }
    if (reinterpret_cast<uintptr_t>(multicast_out) & 15) { set_error("multicast_out is not 16-byte aligned"); return CSPN_ERR_INVALID_ARGUMENT; }
    if (iters == 0) { set_error("the fused gather needs prop_time >= 1"); return CSPN_ERR_UNSUPPORTED; }
    return CSPN_OK;
}

Fan make_fan(float* const* peer_out, int n_peer, float* multicast_out) {
    Fan f{};
    for (int i = 0; i < n_peer; ++i) f.peer[i] = peer_out[i];
    f.n_peer = n_peer;
    f.mc = multicast_out;
    return f;
}

// Picks the algorithm actually run for `algo` on this problem.  AUTO prefers the cluster kernel.
int resolve_algo(const Problem2D& p, int algo, char* why, int why_len, const void* ws = nullptr) {
    if (algo == CSPN_ALGO_GENERIC) return CSPN_ALGO_GENERIC;
    if (cluster2d_supported(p, why, why_len, ws)) return CSPN_ALGO_CLUSTER;
    return algo == CSPN_ALGO_CLUSTER ? (int)CSPN_ERR_UNSUPPORTED : (int)CSPN_ALGO_GENERIC;
}

}  // namespace
}  // namespace cspn

using namespace cspn;

extern "C" {

const char* cspn_last_error(void) { return g_err; }
int cspn_version(void) { return 100; }
int cspn_last_algo(void) { return g_last_algo; }
int cspn_last_launches(void) { return g_last_launches; }

void* cspn_host_alloc(size_t bytes) {
    void* p = nullptr;
    if (cudaHostAlloc(&p, bytes, cudaHostAllocDefault) != cudaSuccess) {
        set_error("cudaHostAlloc(%zu) failed", bytes);
        cudaGetLastError();
        return nullptr;
    }
    return p;
}
void cspn_host_free(void* p) {
    if (p) cudaFreeHost(p);
}

size_t cspn2d_workspace_bytes(int B, int C, int H, int W, int iters, int algo) {
    if (B <= 0 || C <= 0 || H <= 0 || W <= 0 || iters <= 0) return 0;
    if (algo != CSPN_ALGO_GENERIC) {
        Problem2D p{nullptr, nullptr, nullptr, nullptr, B, C, H, W, 8, iters, 0};
        char why[8];
        if (cluster2d_supported(p, why, sizeof(why))) return cluster2d_workspace_bytes(B, C, H, W, iters);
        if (algo == CSPN_ALGO_CLUSTER) return 0;   // the forward call will report why it is unsupported
    }
    return generic2d_workspace_bytes(B, C, H, W, iters);
}

int cspn2d_fwd_f32(const float* guidance, const float* blur, const float* sparse, float* out, int B, int C, int H,
                   int W, int guidance_channels, int iters, int norm_type, int algo, void* workspace,
                   size_t workspace_bytes, cspn_stream_t stream) {
    clear_error();
    g_last_launches = 0;
    int rc = check2d(guidance, blur, out, B, C, H, W, guidance_channels, iters, norm_type, algo);
    if (rc != CSPN_OK) return rc;
    DeviceGuard guard(device_of(blur));
    if (!guard.ok) { set_error("cannot select the device of `blur`"); return CSPN_ERR_CUDA; }
    Problem2D p{guidance, blur, sparse, out, B, C, H, W, guidance_channels, iters, norm_type == CSPN_NORM_8SUM_ABS};
    char why[256] = "";
    const int chosen = (iters == 0) ? CSPN_ALGO_GENERIC : resolve_algo(p, algo, why, sizeof(why), workspace);
    if (chosen < 0) { set_error("cluster kernel unsupported for this problem: %s", why); return chosen; }
    g_last_algo = chosen;
    int launches = 0;
    if (chosen == CSPN_ALGO_GENERIC && algo == CSPN_ALGO_AUTO && iters > 0) {
        // AUTO sized its workspace for the cluster kernel (cspn2d_workspace_bytes cannot see the pointers); when the
        // problem then has to take the generic path, say so instead of a bare "workspace too small"
        const size_t need = generic2d_workspace_bytes(B, C, H, W, iters);
        if (!workspace || workspace_bytes < need) {
            set_error("CSPN_ALGO_AUTO falls back to the generic path here (%s), which needs %zu workspace bytes (got %zu): "
                      "query cspn2d_workspace_bytes(..., CSPN_ALGO_GENERIC) or pass 16-byte aligned tensors and workspace",
                      why[0] ? why : "cluster kernel declined", need, workspace ? workspace_bytes : (size_t)0);
            return CSPN_ERR_WORKSPACE;
        }
    }
    rc = (chosen == CSPN_ALGO_CLUSTER) ? cluster2d_forward(p, workspace, workspace_bytes, (cudaStream_t)stream, &launches)
                                       : generic2d_forward(p, workspace, workspace_bytes, (cudaStream_t)stream, &launches);
    g_last_launches = launches;
    return rc;
}

int cspn2d_fwd_gather_f32(const float* guidance, const float* blur, const float* sparse, float* out, float* const* peer_out,
                          int n_peer, float* multicast_out, int B, int C, int H, int W, int guidance_channels, int iters,
                          int norm_type, void* workspace, size_t workspace_bytes, cspn_stream_t stream) {
    clear_error();
    g_last_launches = 0;
    int rc = check2d(guidance, blur, out, B, C, H, W, guidance_channels, iters, norm_type, CSPN_ALGO_CLUSTER);
    if (rc != CSPN_OK) return rc;
    rc = check_gather(peer_out, n_peer, multicast_out, iters);
    if (rc != CSPN_OK) return rc;
    DeviceGuard guard(device_of(blur));
    if (!guard.ok) { set_error("cannot select the device of `blur`"); return CSPN_ERR_CUDA; }
    Problem2D p{guidance, blur, sparse, out, B, C, H, W, guidance_channels, iters, norm_type == CSPN_NORM_8SUM_ABS};
    char why[256] = "";
    if (!cluster2d_supported(p, why, sizeof(why), workspace)) {
        set_error("the fused gather runs in the cluster kernel's epilogue, which cannot take this problem: %s", why);
        return CSPN_ERR_UNSUPPORTED;
    }
    g_last_algo = CSPN_ALGO_CLUSTER;
    int launches = 0;
    rc = cluster2d_forward(p, workspace, workspace_bytes, (cudaStream_t)stream, &launches, peer_out, n_peer, multicast_out);
    g_last_launches = launches;
    return rc;
}

size_t cspn2d_bwd_workspace_bytes(int B, int C, int H, int W, int iters) {
    if (B <= 0 || C <= 0 || H <= 0 || W <= 0 || iters < 0) return 0;
    return bwd2d_workspace_bytes(B, C, H, W, iters);
}

int cspn2d_bwd_f32(const float* guidance, const float* blur, const float* sparse, const float* grad_out,
                   float* grad_guidance, float* grad_blur, int B, int C, int H, int W, int guidance_channels,
                   int iters, int norm_type, void* workspace, size_t workspace_bytes, cspn_stream_t stream) {
    clear_error();
    g_last_launches = 0;
    float dummy;
    int rc = check2d(guidance, blur, &dummy, B, C, H, W, guidance_channels, iters, norm_type, CSPN_ALGO_AUTO);
    if (rc != CSPN_OK) return rc;
    if (!grad_out) { set_error("null grad_out"); return CSPN_ERR_INVALID_ARGUMENT; }
    DeviceGuard guard(device_of(blur));
    if (!guard.ok) { set_error("cannot select the device of `blur`"); return CSPN_ERR_CUDA; }
    Problem2D p{guidance, blur, sparse, nullptr, B, C, H, W, guidance_channels, iters, norm_type == CSPN_NORM_8SUM_ABS};
    int launches = 0;
    rc = bwd2d(p, grad_out, grad_guidance, grad_blur, workspace, workspace_bytes, (cudaStream_t)stream, &launches);
    g_last_launches = launches;
    return rc;
}

// ---- K x K kernels: K = 3 is the operator above, K = 5 / 7 run in cspn2d_wide.cu ----------------------------------
static bool kernel_size_ok(int K) { return K == 3 || K == 5 || K == 7; }

static int check2d_k(const float* guidance, const float* blur, const void* out, int B, int C, int H, int W, int gch, int K,
                     int iters, int norm_type) {
    if (!guidance || !blur || !out) { set_error("null tensor pointer"); return CSPN_ERR_INVALID_ARGUMENT; }
    if (B <= 0 || C <= 0 || H <= 0 || W <= 0) { set_error("non-positive shape B=%d C=%d H=%d W=%d", B, C, H, W); return CSPN_ERR_INVALID_ARGUMENT; }
    if (!kernel_size_ok(K)) { set_error("kernel size must be 3, 5 or 7, got %d", K); return CSPN_ERR_INVALID_ARGUMENT; }
    if (gch < K * K - 1) { set_error("a %dx%d kernel needs >= %d guidance channels, got %d", K, K, K * K - 1, gch); return CSPN_ERR_INVALID_ARGUMENT; }
    if (iters < 0) { set_error("prop_time must be >= 0, got %d", iters); return CSPN_ERR_INVALID_ARGUMENT; }
    if (norm_type != CSPN_NORM_8SUM && norm_type != CSPN_NORM_8SUM_ABS) { set_error("unknown norm_type %d", norm_type); return CSPN_ERR_INVALID_ARGUMENT; }
    return CSPN_OK;
}

size_t cspn2d_k_workspace_bytes(int B, int C, int H, int W, int K, int iters) {
    if (B <= 0 || C <= 0 || H <= 0 || W <= 0 || iters <= 0 || !kernel_size_ok(K)) return 0;
    if (K == 3) return cspn2d_workspace_bytes(B, C, H, W, iters, CSPN_ALGO_AUTO);
    return widek_workspace_bytes(B, C, H, W, K, iters);
}

int cspn2d_k_fwd_f32(const float* guidance, const float* blur, const float* sparse, float* out, int B, int C, int H, int W,
                     int guidance_channels, int K, int iters, int norm_type, void* workspace, size_t workspace_bytes,
                     cspn_stream_t stream) {
    clear_error();
    g_last_launches = 0;
    int rc = check2d_k(guidance, blur, out, B, C, H, W, guidance_channels, K, iters, norm_type);
    if (rc != CSPN_OK) return rc;
    if (K == 3)
        return cspn2d_fwd_f32(guidance, blur, sparse, out, B, C, H, W, guidance_channels, iters, norm_type, CSPN_ALGO_AUTO,
                              workspace, workspace_bytes, stream);
    DeviceGuard guard(device_of(blur));
    if (!guard.ok) { set_error("cannot select the device of `blur`"); return CSPN_ERR_CUDA; }
    Problem2D p{guidance, blur, sparse, out, B, C, H, W, guidance_channels, iters, norm_type == CSPN_NORM_8SUM_ABS};
    int launches = 0;
    rc = widek_forward(p, K, workspace, workspace_bytes, (cudaStream_t)stream, &launches);
    g_last_launches = launches;
    return rc;
}

int cspn2d_k_fwd_gather_f32(const float* guidance, const float* blur, const float* sparse, float* out, float* const* peer_out,
                            int n_peer, float* multicast_out, int B, int C, int H, int W, int guidance_channels, int K,
                            int iters, int norm_type, void* workspace, size_t workspace_bytes, cspn_stream_t stream) {
    clear_error();
    g_last_launches = 0;
    int rc = check2d_k(guidance, blur, out, B, C, H, W, guidance_channels, K, iters, norm_type);
    if (rc != CSPN_OK) return rc;
    if (K == 3)
        return cspn2d_fwd_gather_f32(guidance, blur, sparse, out, peer_out, n_peer, multicast_out, B, C, H, W,
                                     guidance_channels, iters, norm_type, workspace, workspace_bytes, stream);
    rc = check_gather(peer_out, n_peer, multicast_out, iters);
    if (rc != CSPN_OK) return rc;
    DeviceGuard guard(device_of(blur));
    if (!guard.ok) { set_error("cannot select the device of `blur`"); return CSPN_ERR_CUDA; }
    Problem2D p{guidance, blur, sparse, out, B, C, H, W, guidance_channels, iters, norm_type == CSPN_NORM_8SUM_ABS};
    const Fan fan = make_fan(peer_out, n_peer, multicast_out);
    int launches = 0;
    rc = widek_forward(p, K, workspace, workspace_bytes, (cudaStream_t)stream, &launches, &fan);
    g_last_launches = launches;
    return rc;
}

size_t cspn2d_k_bwd_workspace_bytes(int B, int C, int H, int W, int K, int iters) {
    if (B <= 0 || C <= 0 || H <= 0 || W <= 0 || iters < 0 || !kernel_size_ok(K)) return 0;
    if (K == 3) return cspn2d_bwd_workspace_bytes(B, C, H, W, iters);
    return widek_bwd_workspace_bytes(B, C, H, W, K, iters);
}

int cspn2d_k_bwd_f32(const float* guidance, const float* blur, const float* sparse, const float* grad_out,
                     float* grad_guidance, float* grad_blur, int B, int C, int H, int W, int guidance_channels, int K,
                     int iters, int norm_type, void* workspace, size_t workspace_bytes, cspn_stream_t stream) {
    clear_error();
    g_last_launches = 0;
    int rc = check2d_k(guidance, blur, grad_out, B, C, H, W, guidance_channels, K, iters, norm_type);
    if (rc != CSPN_OK) return rc;
    if (K == 3)
        return cspn2d_bwd_f32(guidance, blur, sparse, grad_out, grad_guidance, grad_blur, B, C, H, W, guidance_channels,
                              iters, norm_type, workspace, workspace_bytes, stream);
    DeviceGuard guard(device_of(blur));
    if (!guard.ok) { set_error("cannot select the device of `blur`"); return CSPN_ERR_CUDA; }
    Problem2D p{guidance, blur, sparse, nullptr, B, C, H, W, guidance_channels, iters, norm_type == CSPN_NORM_8SUM_ABS};
    int launches = 0;
    rc = widek_backward(p, K, grad_out, grad_guidance, grad_blur, workspace, workspace_bytes, (cudaStream_t)stream, &launches);
    g_last_launches = launches;
    return rc;
}

// ---- 2D 'paddle' (own-location norm), K in {3, 5, 7}: every K in cspn2d_wide.cu ------------------------------------
static int check2d_paddle(const float* guidance, const float* feat, const void* out, int B, int C, int H, int W, int K,
                          int iters) {
    if (!guidance || !feat || !out) { set_error("null tensor pointer"); return CSPN_ERR_INVALID_ARGUMENT; }
    if (B <= 0 || C <= 0 || H <= 0 || W <= 0) { set_error("non-positive shape B=%d C=%d H=%d W=%d", B, C, H, W); return CSPN_ERR_INVALID_ARGUMENT; }
    if (!kernel_size_ok(K)) { set_error("kernel size must be 3, 5 or 7, got %d", K); return CSPN_ERR_INVALID_ARGUMENT; }
    if (iters < 0) { set_error("prop_time must be >= 0, got %d", iters); return CSPN_ERR_INVALID_ARGUMENT; }
    return CSPN_OK;
}

size_t cspn2d_paddle_workspace_bytes(int B, int C, int H, int W, int K, int iters) {
    if (B <= 0 || C <= 0 || H <= 0 || W <= 0 || iters <= 0 || !kernel_size_ok(K)) return 0;
    return widek_workspace_bytes(B, C, H, W, K, iters);
}

int cspn2d_paddle_fwd_f32(const float* guidance, const float* feat, float* out, int B, int C, int H, int W, int K, int iters,
                          void* workspace, size_t workspace_bytes, cspn_stream_t stream) {
    clear_error();
    g_last_launches = 0;
    int rc = check2d_paddle(guidance, feat, out, B, C, H, W, K, iters);
    if (rc != CSPN_OK) return rc;
    DeviceGuard guard(device_of(feat));
    if (!guard.ok) { set_error("cannot select the device of `feat`"); return CSPN_ERR_CUDA; }
    Problem2D p{guidance, feat, nullptr, out, B, C, H, W, K * K - 1, iters, 0};
    int launches = 0;
    rc = widek_paddle_forward(p, K, workspace, workspace_bytes, (cudaStream_t)stream, &launches);
    g_last_launches = launches;
    return rc;
}

int cspn2d_paddle_fwd_gather_f32(const float* guidance, const float* feat, float* out, float* const* peer_out, int n_peer,
                                 float* multicast_out, int B, int C, int H, int W, int K, int iters, void* workspace,
                                 size_t workspace_bytes, cspn_stream_t stream) {
    clear_error();
    g_last_launches = 0;
    int rc = check2d_paddle(guidance, feat, out, B, C, H, W, K, iters);
    if (rc != CSPN_OK) return rc;
    rc = check_gather(peer_out, n_peer, multicast_out, iters);
    if (rc != CSPN_OK) return rc;
    DeviceGuard guard(device_of(feat));
    if (!guard.ok) { set_error("cannot select the device of `feat`"); return CSPN_ERR_CUDA; }
    Problem2D p{guidance, feat, nullptr, out, B, C, H, W, K * K - 1, iters, 0};
    const Fan fan = make_fan(peer_out, n_peer, multicast_out);
    int launches = 0;
    rc = widek_paddle_forward(p, K, workspace, workspace_bytes, (cudaStream_t)stream, &launches, &fan);
    g_last_launches = launches;
    return rc;
}

size_t cspn2d_paddle_bwd_workspace_bytes(int B, int C, int H, int W, int K, int iters) {
    if (B <= 0 || C <= 0 || H <= 0 || W <= 0 || iters <= 0 || !kernel_size_ok(K)) return 0;
    return widek_bwd_workspace_bytes(B, C, H, W, K, iters);
}

int cspn2d_paddle_bwd_f32(const float* guidance, const float* feat, const float* grad_out, float* grad_guidance, float* grad_feat,
                          int B, int C, int H, int W, int K, int iters, void* workspace, size_t workspace_bytes,
                          cspn_stream_t stream) {
    clear_error();
    g_last_launches = 0;
    int rc = check2d_paddle(guidance, feat, grad_out, B, C, H, W, K, iters);
    if (rc != CSPN_OK) return rc;
    DeviceGuard guard(device_of(feat));
    if (!guard.ok) { set_error("cannot select the device of `feat`"); return CSPN_ERR_CUDA; }
    Problem2D p{guidance, feat, nullptr, nullptr, B, C, H, W, K * K - 1, iters, 0};
    int launches = 0;
    rc = widek_paddle_backward(p, K, grad_out, grad_guidance, grad_feat, workspace, workspace_bytes, (cudaStream_t)stream,
                               &launches);
    g_last_launches = launches;
    return rc;
}

size_t cspn3d_workspace_bytes(int B, int C, int D, int H, int W, int iters) {
    if (B <= 0 || C <= 0 || D <= 0 || H <= 0 || W <= 0 || iters <= 0) return 0;
    return generic3d_workspace_bytes(B, C, D, H, W, iters);
}

static int check3d(const float* guidance, const float* feat, const float* out, int B, int C, int D, int H, int W, int iters,
                   int norm_type) {
    if (!guidance || !feat || !out) { set_error("null tensor pointer"); return CSPN_ERR_INVALID_ARGUMENT; }
    if (B <= 0 || C <= 0 || D <= 0 || H <= 0 || W <= 0) { set_error("non-positive shape"); return CSPN_ERR_INVALID_ARGUMENT; }
    if (iters < 0) { set_error("prop_step must be >= 0"); return CSPN_ERR_INVALID_ARGUMENT; }
    if (norm_type < CSPN_NORM_26SUM || norm_type > CSPN_NORM_PADDLE) { set_error("unknown 3D norm_type %d", norm_type); return CSPN_ERR_INVALID_ARGUMENT; }
    return CSPN_OK;
}

int cspn3d_fwd_f32(const float* guidance, const float* feat, float* out, int B, int C, int D, int H, int W, int iters,
                   int norm_type, void* workspace, size_t workspace_bytes, cspn_stream_t stream) {
    clear_error();
    g_last_launches = 0;
    int rc = check3d(guidance, feat, out, B, C, D, H, W, iters, norm_type);
    if (rc != CSPN_OK) return rc;
    DeviceGuard guard(device_of(feat));
    if (!guard.ok) { set_error("cannot select the device of `feat`"); return CSPN_ERR_CUDA; }
    int launches = 0;
    rc = generic3d_forward(guidance, feat, out, B, C, D, H, W, iters, norm_type, workspace, workspace_bytes,
                           (cudaStream_t)stream, &launches);
    g_last_launches = launches;
    return rc;
}

int cspn3d_fwd_gather_f32(const float* guidance, const float* feat, float* out, float* const* peer_out, int n_peer,
                          float* multicast_out, int B, int C, int D, int H, int W, int iters, int norm_type, void* workspace,
                          size_t workspace_bytes, cspn_stream_t stream) {
    clear_error();
    g_last_launches = 0;
    int rc = check3d(guidance, feat, out, B, C, D, H, W, iters, norm_type);
    if (rc != CSPN_OK) return rc;
    rc = check_gather(peer_out, n_peer, multicast_out, iters);
    if (rc != CSPN_OK) return rc;
    DeviceGuard guard(device_of(feat));
    if (!guard.ok) { set_error("cannot select the device of `feat`"); return CSPN_ERR_CUDA; }
    const Fan fan = make_fan(peer_out, n_peer, multicast_out);
    int launches = 0;
    rc = generic3d_forward(guidance, feat, out, B, C, D, H, W, iters, norm_type, workspace, workspace_bytes,
                           (cudaStream_t)stream, &launches, &fan);
    g_last_launches = launches;
    return rc;
}

size_t cspn3d_bwd_workspace_bytes(int B, int C, int D, int H, int W, int iters) {
    if (B <= 0 || C <= 0 || D <= 0 || H <= 0 || W <= 0 || iters <= 0) return 0;
    return bwd3d_workspace_bytes(C, D, H, W, iters);
}

int cspn3d_bwd_f32(const float* guidance, const float* feat, const float* grad_out, float* grad_guidance, float* grad_feat,
                   int B, int C, int D, int H, int W, int iters, int norm_type, void* workspace, size_t workspace_bytes,
                   cspn_stream_t stream) {
    clear_error();
    g_last_launches = 0;
    if (!guidance || !feat || !grad_out) { set_error("null tensor pointer"); return CSPN_ERR_INVALID_ARGUMENT; }
    if (B <= 0 || C <= 0 || D <= 0 || H <= 0 || W <= 0 || iters < 0) { set_error("invalid 3D shape / prop_step"); return CSPN_ERR_INVALID_ARGUMENT; }
    if (norm_type < CSPN_NORM_26SUM || norm_type > CSPN_NORM_PADDLE) { set_error("unknown 3D norm_type %d", norm_type); return CSPN_ERR_INVALID_ARGUMENT; }
    DeviceGuard guard(device_of(feat));
    if (!guard.ok) { set_error("cannot select the device of `feat`"); return CSPN_ERR_CUDA; }
    int launches = 0;
    int rc = bwd3d(guidance, feat, grad_out, grad_guidance, grad_feat, B, C, D, H, W, iters, norm_type, workspace, workspace_bytes,
                   (cudaStream_t)stream, &launches);
    g_last_launches = launches;
    return rc;
}

// ---- K x K x K kernels: K = 3 is the 3D operator above, K = 5 runs in cspn3d_wide.cu ------------------------------
static int check3d_k(const float* guidance, const float* feat, const void* out, int B, int C, int D, int H, int W, int K,
                     int iters, int norm_type) {
    if (!guidance || !feat || !out) { set_error("null tensor pointer"); return CSPN_ERR_INVALID_ARGUMENT; }
    if (B <= 0 || C <= 0 || D <= 0 || H <= 0 || W <= 0) { set_error("non-positive shape B=%d C=%d D=%d H=%d W=%d", B, C, D, H, W); return CSPN_ERR_INVALID_ARGUMENT; }
    if (K != 3 && K != 5) { set_error("3D kernel size must be 3 or 5, got %d", K); return CSPN_ERR_INVALID_ARGUMENT; }
    if (iters < 0) { set_error("prop_time must be >= 0, got %d", iters); return CSPN_ERR_INVALID_ARGUMENT; }
    if (norm_type < CSPN_NORM_26SUM || norm_type > CSPN_NORM_PADDLE) { set_error("unknown 3D norm_type %d", norm_type); return CSPN_ERR_INVALID_ARGUMENT; }
    return CSPN_OK;
}

size_t cspn3d_k_workspace_bytes(int B, int C, int D, int H, int W, int K, int iters) {
    if (B <= 0 || C <= 0 || D <= 0 || H <= 0 || W <= 0 || iters <= 0 || (K != 3 && K != 5)) return 0;
    if (K == 3) return cspn3d_workspace_bytes(B, C, D, H, W, iters);
    return widek3d_workspace_bytes(B, C, D, H, W, K, iters);
}

int cspn3d_k_fwd_f32(const float* guidance, const float* feat, float* out, int B, int C, int D, int H, int W, int K, int iters,
                     int norm_type, void* workspace, size_t workspace_bytes, cspn_stream_t stream) {
    clear_error();
    g_last_launches = 0;
    int rc = check3d_k(guidance, feat, out, B, C, D, H, W, K, iters, norm_type);
    if (rc != CSPN_OK) return rc;
    if (K == 3) return cspn3d_fwd_f32(guidance, feat, out, B, C, D, H, W, iters, norm_type, workspace, workspace_bytes, stream);
    DeviceGuard guard(device_of(feat));
    if (!guard.ok) { set_error("cannot select the device of `feat`"); return CSPN_ERR_CUDA; }
    int launches = 0;
    rc = widek3d_forward(guidance, feat, out, B, C, D, H, W, K, iters, norm_type, workspace, workspace_bytes, (cudaStream_t)stream,
                         &launches);
    g_last_launches = launches;
    return rc;
}

int cspn3d_k_fwd_gather_f32(const float* guidance, const float* feat, float* out, float* const* peer_out, int n_peer,
                            float* multicast_out, int B, int C, int D, int H, int W, int K, int iters, int norm_type,
                            void* workspace, size_t workspace_bytes, cspn_stream_t stream) {
    clear_error();
    g_last_launches = 0;
    int rc = check3d_k(guidance, feat, out, B, C, D, H, W, K, iters, norm_type);
    if (rc != CSPN_OK) return rc;
    if (K == 3)
        return cspn3d_fwd_gather_f32(guidance, feat, out, peer_out, n_peer, multicast_out, B, C, D, H, W, iters, norm_type,
                                     workspace, workspace_bytes, stream);
    rc = check_gather(peer_out, n_peer, multicast_out, iters);
    if (rc != CSPN_OK) return rc;
    DeviceGuard guard(device_of(feat));
    if (!guard.ok) { set_error("cannot select the device of `feat`"); return CSPN_ERR_CUDA; }
    const Fan fan = make_fan(peer_out, n_peer, multicast_out);
    int launches = 0;
    rc = widek3d_forward(guidance, feat, out, B, C, D, H, W, K, iters, norm_type, workspace, workspace_bytes, (cudaStream_t)stream,
                         &launches, &fan);
    g_last_launches = launches;
    return rc;
}

size_t cspn3d_k_bwd_workspace_bytes(int B, int C, int D, int H, int W, int K, int iters) {
    if (B <= 0 || C <= 0 || D <= 0 || H <= 0 || W <= 0 || iters <= 0 || (K != 3 && K != 5)) return 0;
    if (K == 3) return cspn3d_bwd_workspace_bytes(B, C, D, H, W, iters);
    return widek3d_bwd_workspace_bytes(C, D, H, W, K, iters);
}

int cspn3d_k_bwd_f32(const float* guidance, const float* feat, const float* grad_out, float* grad_guidance, float* grad_feat,
                     int B, int C, int D, int H, int W, int K, int iters, int norm_type, void* workspace, size_t workspace_bytes,
                     cspn_stream_t stream) {
    clear_error();
    g_last_launches = 0;
    int rc = check3d_k(guidance, feat, grad_out, B, C, D, H, W, K, iters, norm_type);
    if (rc != CSPN_OK) return rc;
    if (K == 3)
        return cspn3d_bwd_f32(guidance, feat, grad_out, grad_guidance, grad_feat, B, C, D, H, W, iters, norm_type, workspace,
                              workspace_bytes, stream);
    DeviceGuard guard(device_of(feat));
    if (!guard.ok) { set_error("cannot select the device of `feat`"); return CSPN_ERR_CUDA; }
    int launches = 0;
    rc = widek3d_backward(guidance, feat, grad_out, grad_guidance, grad_feat, B, C, D, H, W, K, iters, norm_type, workspace,
                          workspace_bytes, (cudaStream_t)stream, &launches);
    g_last_launches = launches;
    return rc;
}

// ---- caller-supplied gates (fluid.layers.affinity_propagate): 2D K in {3, 5, 7}, 3D K in {3, 5} ----------------------
static int check_gates(const float* gates, const float* feat, const void* out, int B, int C, int D, int H, int W, int K,
                       int iters, bool is3d) {
    if (!gates || !feat || !out) { set_error("null tensor pointer"); return CSPN_ERR_INVALID_ARGUMENT; }
    if (B <= 0 || C <= 0 || D <= 0 || H <= 0 || W <= 0) { set_error("non-positive shape B=%d C=%d D=%d H=%d W=%d", B, C, D, H, W); return CSPN_ERR_INVALID_ARGUMENT; }
    if (is3d ? (K != 3 && K != 5) : !kernel_size_ok(K)) { set_error("%s kernel size must be %s, got %d", is3d ? "3D" : "2D", is3d ? "3 or 5" : "3, 5 or 7", K); return CSPN_ERR_INVALID_ARGUMENT; }
    if (iters < 0) { set_error("prop_step must be >= 0, got %d", iters); return CSPN_ERR_INVALID_ARGUMENT; }
    return CSPN_OK;
}

size_t cspn2d_gates_workspace_bytes(int B, int C, int H, int W, int K, int iters) {
    if (B <= 0 || C <= 0 || H <= 0 || W <= 0 || iters <= 0 || !kernel_size_ok(K)) return 0;
    return widek_gates_workspace_bytes(B, C, H, W, iters);
}

int cspn2d_gates_fwd_f32(const float* gates, const float* feat, float* out, int B, int C, int H, int W, int K, int iters,
                         void* workspace, size_t workspace_bytes, cspn_stream_t stream) {
    clear_error();
    g_last_launches = 0;
    int rc = check_gates(gates, feat, out, B, C, 1, H, W, K, iters, false);
    if (rc != CSPN_OK) return rc;
    DeviceGuard guard(device_of(feat));
    if (!guard.ok) { set_error("cannot select the device of `feat`"); return CSPN_ERR_CUDA; }
    Problem2D p{gates, feat, nullptr, out, B, C, H, W, K * K - 1, iters, 0};
    int launches = 0;
    rc = widek_gates_forward(p, K, workspace, workspace_bytes, (cudaStream_t)stream, &launches);
    g_last_launches = launches;
    return rc;
}

int cspn2d_gates_fwd_gather_f32(const float* gates, const float* feat, float* out, float* const* peer_out, int n_peer,
                                float* multicast_out, int B, int C, int H, int W, int K, int iters, void* workspace,
                                size_t workspace_bytes, cspn_stream_t stream) {
    clear_error();
    g_last_launches = 0;
    int rc = check_gates(gates, feat, out, B, C, 1, H, W, K, iters, false);
    if (rc != CSPN_OK) return rc;
    rc = check_gather(peer_out, n_peer, multicast_out, iters);
    if (rc != CSPN_OK) return rc;
    DeviceGuard guard(device_of(feat));
    if (!guard.ok) { set_error("cannot select the device of `feat`"); return CSPN_ERR_CUDA; }
    Problem2D p{gates, feat, nullptr, out, B, C, H, W, K * K - 1, iters, 0};
    const Fan fan = make_fan(peer_out, n_peer, multicast_out);
    int launches = 0;
    rc = widek_gates_forward(p, K, workspace, workspace_bytes, (cudaStream_t)stream, &launches, &fan);
    g_last_launches = launches;
    return rc;
}

size_t cspn2d_gates_bwd_workspace_bytes(int B, int C, int H, int W, int K, int iters) {
    if (B <= 0 || C <= 0 || H <= 0 || W <= 0 || iters <= 0 || !kernel_size_ok(K)) return 0;
    return widek_gates_bwd_workspace_bytes(B, C, H, W, iters);
}

int cspn2d_gates_bwd_f32(const float* gates, const float* feat, const float* grad_out, float* grad_gates, float* grad_feat,
                         int B, int C, int H, int W, int K, int iters, void* workspace, size_t workspace_bytes,
                         cspn_stream_t stream) {
    clear_error();
    g_last_launches = 0;
    int rc = check_gates(gates, feat, grad_out, B, C, 1, H, W, K, iters, false);
    if (rc != CSPN_OK) return rc;
    DeviceGuard guard(device_of(feat));
    if (!guard.ok) { set_error("cannot select the device of `feat`"); return CSPN_ERR_CUDA; }
    Problem2D p{gates, feat, nullptr, nullptr, B, C, H, W, K * K - 1, iters, 0};
    int launches = 0;
    rc = widek_gates_backward(p, K, grad_out, grad_gates, grad_feat, workspace, workspace_bytes, (cudaStream_t)stream, &launches);
    g_last_launches = launches;
    return rc;
}

size_t cspn3d_gates_workspace_bytes(int B, int C, int D, int H, int W, int K, int iters) {
    if (B <= 0 || C <= 0 || D <= 0 || H <= 0 || W <= 0 || iters <= 0 || (K != 3 && K != 5)) return 0;
    return widek3d_gates_workspace_bytes(B, C, D, H, W, iters);
}

int cspn3d_gates_fwd_f32(const float* gates, const float* feat, float* out, int B, int C, int D, int H, int W, int K, int iters,
                         void* workspace, size_t workspace_bytes, cspn_stream_t stream) {
    clear_error();
    g_last_launches = 0;
    int rc = check_gates(gates, feat, out, B, C, D, H, W, K, iters, true);
    if (rc != CSPN_OK) return rc;
    DeviceGuard guard(device_of(feat));
    if (!guard.ok) { set_error("cannot select the device of `feat`"); return CSPN_ERR_CUDA; }
    int launches = 0;
    rc = widek3d_gates_forward(gates, feat, out, B, C, D, H, W, K, iters, workspace, workspace_bytes, (cudaStream_t)stream, &launches);
    g_last_launches = launches;
    return rc;
}

int cspn3d_gates_fwd_gather_f32(const float* gates, const float* feat, float* out, float* const* peer_out, int n_peer,
                                float* multicast_out, int B, int C, int D, int H, int W, int K, int iters, void* workspace,
                                size_t workspace_bytes, cspn_stream_t stream) {
    clear_error();
    g_last_launches = 0;
    int rc = check_gates(gates, feat, out, B, C, D, H, W, K, iters, true);
    if (rc != CSPN_OK) return rc;
    rc = check_gather(peer_out, n_peer, multicast_out, iters);
    if (rc != CSPN_OK) return rc;
    DeviceGuard guard(device_of(feat));
    if (!guard.ok) { set_error("cannot select the device of `feat`"); return CSPN_ERR_CUDA; }
    const Fan fan = make_fan(peer_out, n_peer, multicast_out);
    int launches = 0;
    rc = widek3d_gates_forward(gates, feat, out, B, C, D, H, W, K, iters, workspace, workspace_bytes, (cudaStream_t)stream,
                               &launches, &fan);
    g_last_launches = launches;
    return rc;
}

size_t cspn3d_gates_bwd_workspace_bytes(int B, int C, int D, int H, int W, int K, int iters) {
    if (B <= 0 || C <= 0 || D <= 0 || H <= 0 || W <= 0 || iters <= 0 || (K != 3 && K != 5)) return 0;
    return widek3d_gates_bwd_workspace_bytes(C, D, H, W, iters);
}

int cspn3d_gates_bwd_f32(const float* gates, const float* feat, const float* grad_out, float* grad_gates, float* grad_feat,
                         int B, int C, int D, int H, int W, int K, int iters, void* workspace, size_t workspace_bytes,
                         cspn_stream_t stream) {
    clear_error();
    g_last_launches = 0;
    int rc = check_gates(gates, feat, grad_out, B, C, D, H, W, K, iters, true);
    if (rc != CSPN_OK) return rc;
    DeviceGuard guard(device_of(feat));
    if (!guard.ok) { set_error("cannot select the device of `feat`"); return CSPN_ERR_CUDA; }
    int launches = 0;
    rc = widek3d_gates_backward(gates, feat, grad_out, grad_gates, grad_feat, B, C, D, H, W, K, iters, workspace, workspace_bytes,
                                (cudaStream_t)stream, &launches);
    g_last_launches = launches;
    return rc;
}

// ---- unpool + crop + 3x3 convolution (the guidance and depth heads) ---------------------------------------------------
static int check_unpool_conv(const void* x, const void* weight, const void* out, int B, int Cin, int h, int w, int Cout, int H,
                             int W) {
    if (!x || !weight || !out) { set_error("null tensor pointer"); return CSPN_ERR_INVALID_ARGUMENT; }
    if (B <= 0 || Cin <= 0 || h <= 0 || w <= 0 || Cout <= 0 || H <= 0 || W <= 0) {
        set_error("non-positive size B=%d Cin=%d h=%d w=%d Cout=%d H=%d W=%d", B, Cin, h, w, Cout, H, W);
        return CSPN_ERR_INVALID_ARGUMENT;
    }
    if (H > 2 * h || W > 2 * w) { set_error("output %dx%d exceeds the unpooled map %dx%d", H, W, 2 * h, 2 * w); return CSPN_ERR_INVALID_ARGUMENT; }
    if ((reinterpret_cast<uintptr_t>(x) | reinterpret_cast<uintptr_t>(weight) | reinterpret_cast<uintptr_t>(out)) & 3) {
        set_error("tensor pointers must be 4-byte aligned");
        return CSPN_ERR_INVALID_ARGUMENT;
    }
    const char* why = "";
    if (!unpool_conv_launchable(B, Cin, Cout, &why)) { set_error("the launch grid cannot take this shape: %s", why); return CSPN_ERR_UNSUPPORTED; }
    return CSPN_OK;
}

int cspn_unpool_conv3x3_fwd_f32(const float* x, const float* weight, float* out, int B, int Cin, int h, int w, int Cout, int H,
                                int W, cspn_stream_t stream) {
    clear_error();
    g_last_launches = 0;
    int rc = check_unpool_conv(x, weight, out, B, Cin, h, w, Cout, H, W);
    if (rc != CSPN_OK) return rc;
    DeviceGuard guard(device_of(x));
    if (!guard.ok) { set_error("cannot select the device of `x`"); return CSPN_ERR_CUDA; }
    int launches = 0;
    rc = unpool_conv_forward(x, weight, out, B, Cin, h, w, Cout, H, W, (cudaStream_t)stream, &launches);
    g_last_launches = launches;
    return rc;
}

size_t cspn_unpool_conv3x3_bwd_workspace_bytes(int B, int Cin, int h, int w, int Cout, int H, int W) {
    if (B <= 0 || Cin <= 0 || h <= 0 || w <= 0 || Cout <= 0 || H <= 0 || W <= 0 || H > 2 * h || W > 2 * w) return 0;
    return unpool_conv_bwd_workspace_bytes(B, Cin, H, W, Cout);
}

int cspn_unpool_conv3x3_bwd_f32(const float* x, const float* weight, const float* grad_out, float* grad_x, float* grad_weight,
                                int B, int Cin, int h, int w, int Cout, int H, int W, void* workspace, size_t workspace_bytes,
                                cspn_stream_t stream) {
    clear_error();
    g_last_launches = 0;
    int rc = check_unpool_conv(x, weight, grad_out, B, Cin, h, w, Cout, H, W);
    if (rc != CSPN_OK) return rc;
    if ((reinterpret_cast<uintptr_t>(grad_x) | reinterpret_cast<uintptr_t>(grad_weight)) & 3) {
        set_error("gradient pointers must be 4-byte aligned");
        return CSPN_ERR_INVALID_ARGUMENT;
    }
    if (grad_weight) {
        const size_t need = unpool_conv_bwd_workspace_bytes(B, Cin, H, W, Cout);
        if (!workspace || workspace_bytes < need || (reinterpret_cast<uintptr_t>(workspace) & 3)) {
            set_error("grad_weight needs %zu bytes of 4-byte aligned workspace (got %zu)", need, workspace_bytes);
            return CSPN_ERR_WORKSPACE;
        }
    }
    DeviceGuard guard(device_of(x));
    if (!guard.ok) { set_error("cannot select the device of `x`"); return CSPN_ERR_CUDA; }
    int launches = 0;
    rc = unpool_conv_backward(x, weight, grad_out, grad_x, grad_weight, B, Cin, h, w, Cout, H, W, workspace, (cudaStream_t)stream,
                              &launches);
    g_last_launches = launches;
    return rc;
}

int cspn2d_describe_plan(int B, int C, int H, int W, int iters, int algo, char* buf, int buf_len) {
    if (!buf || buf_len <= 0) return 0;
    Problem2D p{nullptr, nullptr, nullptr, nullptr, B, C, H, W, 8, iters, 0};
    char why[256] = "";
    const int chosen = resolve_algo(p, algo, why, sizeof(why));
    if (chosen == CSPN_ALGO_CLUSTER) return cluster2d_describe(B, C, H, W, iters, buf, buf_len);
    if (chosen < 0) return snprintf(buf, buf_len, "unsupported: %s", why);
    return snprintf(buf, buf_len, "generic: prep + %d stencil launches, workspace %zu B%s%s", iters,
                    generic2d_workspace_bytes(B, C, H, W, iters), why[0] ? "; cluster kernel not used: " : "", why);
}

int cspn2d_plan_json(int H, int W, int iters, char* buf, int buf_len) {
    if (!buf || buf_len <= 0) return 0;
    if (H <= 0 || W <= 0 || iters <= 0) return snprintf(buf, buf_len, "{\"supported\": false, \"why\": \"invalid shape\"}");
    return cluster2d_plan_json(H, W, iters, 0, buf, buf_len);
}

int cspn2d_plan_json_chained(int H, int W, int iters, char* buf, int buf_len) {
    if (!buf || buf_len <= 0) return 0;
    if (H <= 0 || W <= 0 || iters <= 0) return snprintf(buf, buf_len, "{\"supported\": false, \"why\": \"invalid shape\"}");
    return cluster2d_plan_json(H, W, iters, 1, buf, buf_len);
}

}  // extern "C"

// ---- host-buffer pipeline -------------------------------------------------------------------
// The reference-facing call with HOST buffers (bench.py "e2e"): batch chunks flow through three
// slots, each with its own stream and device buffers, so chunk i's H2D overlaps chunk i-1's kernel;
// results stay on the device and leave in one D2H at the end (see the comment in the 2D entry point).
namespace cspn {
namespace {

struct Slot {
    cudaStream_t stream = nullptr;
    char* buf = nullptr;
    size_t cap = 0;
};
struct HostPipe {
    std::mutex mu;
    Slot slots[3];
    Slot result;          // whole-batch output on the device + the stream of the single D2H at the end
    cudaEvent_t done[3] = {nullptr, nullptr, nullptr};
    int device = -1;
};
HostPipe g_pipes[16];

int ensure_slot(Slot& s, size_t bytes) {
    if (!s.stream) CSPN_CUDA_TRY(cudaStreamCreateWithFlags(&s.stream, cudaStreamNonBlocking));
    if (s.cap < bytes) {
        if (s.buf) CSPN_CUDA_TRY(cudaFree(s.buf));
        s.buf = nullptr;
        s.cap = 0;
        CSPN_CUDA_TRY(cudaMalloc(&s.buf, bytes));
        s.cap = bytes;
    }
    return CSPN_OK;
}

inline size_t align_up(size_t v, size_t a) { return (v + a - 1) / a * a; }

// A host-buffer call that fails half way must not return while earlier chunks' copies and kernels still read the
// caller's buffers or write the pipeline's: on every exit path that did not reach the final synchronisation, drain.
struct DrainOnExit {
    HostPipe& pipe;
    bool armed = true;
    explicit DrainOnExit(HostPipe& p) : pipe(p) {}
    ~DrainOnExit() {
        if (!armed) return;
        for (auto& s : pipe.slots)
            if (s.stream) cudaStreamSynchronize(s.stream);
        if (pipe.result.stream) cudaStreamSynchronize(pipe.result.stream);
        cudaGetLastError();    // the status the caller sees is the one already recorded
    }
};

}  // namespace
}  // namespace cspn

extern "C" CSPN_API int cspn2d_fwd_f32_host(const float* guidance, const float* blur, const float* sparse, float* out, int B,
                                   int C, int H, int W, int guidance_channels, int iters, int norm_type, int algo,
                                   int device) {
    clear_error();
    g_last_launches = 0;
    int rc = check2d(guidance, blur, out, B, C, H, W, guidance_channels, iters, norm_type, algo);
    if (rc != CSPN_OK) return rc;
    if (device < 0 || device >= 16) { set_error("device %d out of range", device); return CSPN_ERR_INVALID_ARGUMENT; }
    DeviceGuard guard(device);
    if (!guard.ok) { set_error("cannot select device %d", device); return CSPN_ERR_CUDA; }
    HostPipe& pipe = g_pipes[device];
    std::lock_guard<std::mutex> lock(pipe.mu);
    DrainOnExit drain(pipe);

    const size_t HW = (size_t)H * W;
    // chunk: about 48 MB of input per slot keeps PCIe transfers long and the kernel grid full
    const size_t per_img = (8 + C + (sparse ? 1 : 0)) * HW * sizeof(float);
    // developer hook for tuning runs: CSPN_B200_HOST_CHUNK_MB overrides the chunk size
    const char* chunk_env = getenv("CSPN_B200_HOST_CHUNK_MB");
    const size_t chunk_bytes = (size_t)(chunk_env && atoi(chunk_env) > 0 ? atoi(chunk_env) : 48) << 20;
    int nb = (int)(chunk_bytes / per_img);
    if (nb < 1) nb = 1;
    if (nb > B) nb = B;
    // keep at least 3 chunks in flight when the batch allows it
    if (B >= 3 && (B + nb - 1) / nb < 3) nb = (B + 2) / 3;

    const size_t g_bytes = align_up((size_t)nb * 8 * HW * sizeof(float), 256);
    const size_t d_bytes = align_up((size_t)nb * C * HW * sizeof(float), 256);
    const size_t s_bytes = sparse ? align_up((size_t)nb * HW * sizeof(float), 256) : 0;
    const size_t ws_bytes = align_up(cspn2d_workspace_bytes(nb, C, H, W, iters, algo), 256);
    const size_t slot_bytes = g_bytes + d_bytes + s_bytes + ws_bytes;
    // Results stay on the device until every chunk has been uploaded: an H2D and a D2H running concurrently share the
    // host link, and the output is only 1/10 of the input, so one D2H at the end beats overlapping it.
    rc = ensure_slot(pipe.result, (size_t)B * C * HW * sizeof(float));
    if (rc != CSPN_OK) return rc;
    float* dout_all = reinterpret_cast<float*>(pipe.result.buf);
    for (auto& e : pipe.done)
        if (!e) CSPN_CUDA_TRY(cudaEventCreateWithFlags(&e, cudaEventDisableTiming));
    const char* ns_env = getenv("CSPN_B200_HOST_STREAMS");   // developer hook for tuning runs
    const int nslots = ns_env && atoi(ns_env) >= 1 && atoi(ns_env) <= 3 ? atoi(ns_env) : 3;
    int launches = 0, chunk = 0;
    for (int b0 = 0; b0 < B; b0 += nb, ++chunk) {
        Slot& s = pipe.slots[chunk % nslots];
        rc = ensure_slot(s, slot_bytes);
        if (rc != CSPN_OK) return rc;
        const int n = (B - b0 < nb) ? B - b0 : nb;
        float* dg = reinterpret_cast<float*>(s.buf);
        float* dd = reinterpret_cast<float*>(s.buf + g_bytes);
        float* dsp = sparse ? reinterpret_cast<float*>(s.buf + g_bytes + d_bytes) : nullptr;
        void* dws = ws_bytes ? s.buf + g_bytes + d_bytes + s_bytes : nullptr;
        // only channels 0..7 of the guidance are used (cspn.py:91-98): copy just those planes, with one linear copy
        // when the guidance has exactly 8 channels.
        if (guidance_channels == 8)
            CSPN_CUDA_TRY(cudaMemcpyAsync(dg, guidance + (size_t)b0 * 8 * HW, (size_t)n * 8 * HW * sizeof(float),
                                          cudaMemcpyHostToDevice, s.stream));
        else
            for (int i = 0; i < n; ++i)
                CSPN_CUDA_TRY(cudaMemcpyAsync(dg + (size_t)i * 8 * HW, guidance + (size_t)(b0 + i) * guidance_channels * HW,
                                              8 * HW * sizeof(float), cudaMemcpyHostToDevice, s.stream));
        CSPN_CUDA_TRY(cudaMemcpyAsync(dd, blur + (size_t)b0 * C * HW, (size_t)n * C * HW * sizeof(float),
                                      cudaMemcpyHostToDevice, s.stream));
        if (sparse)
            CSPN_CUDA_TRY(cudaMemcpyAsync(dsp, sparse + (size_t)b0 * HW, (size_t)n * HW * sizeof(float),
                                          cudaMemcpyHostToDevice, s.stream));
        rc = cspn2d_fwd_f32(dg, dd, dsp, dout_all + (size_t)b0 * C * HW, n, C, H, W, 8, iters, norm_type, algo, dws, ws_bytes,
                            (cspn_stream_t)s.stream);
        if (rc != CSPN_OK) return rc;
        launches += g_last_launches;
    }
    for (int i = 0; i < 3; ++i)
        if (pipe.slots[i].stream) {
            CSPN_CUDA_TRY(cudaEventRecord(pipe.done[i], pipe.slots[i].stream));
            CSPN_CUDA_TRY(cudaStreamWaitEvent(pipe.result.stream, pipe.done[i], 0));
        }
    CSPN_CUDA_TRY(cudaMemcpyAsync(out, dout_all, (size_t)B * C * HW * sizeof(float), cudaMemcpyDeviceToHost, pipe.result.stream));
    CSPN_CUDA_TRY(cudaStreamSynchronize(pipe.result.stream));
    drain.armed = false;
    g_last_launches = launches;
    return CSPN_OK;
}

extern "C" CSPN_API int cspn3d_fwd_f32_host(const float* guidance, const float* feat, float* out, int B, int C, int D, int H,
                                   int W, int iters, int norm_type, int device) {
    clear_error();
    g_last_launches = 0;
    if (!guidance || !feat || !out || B <= 0 || C <= 0 || D <= 0 || H <= 0 || W <= 0 || iters < 0) {
        set_error("invalid 3D arguments");
        return CSPN_ERR_INVALID_ARGUMENT;
    }
    if (device < 0 || device >= 16) { set_error("device %d out of range", device); return CSPN_ERR_INVALID_ARGUMENT; }
    DeviceGuard guard(device);
    if (!guard.ok) { set_error("cannot select device %d", device); return CSPN_ERR_CUDA; }
    HostPipe& pipe = g_pipes[device];
    std::lock_guard<std::mutex> lock(pipe.mu);
    DrainOnExit drain(pipe);
    const size_t V = (size_t)D * H * W;
    const size_t g_bytes = align_up(26 * V * sizeof(float), 256);
    const size_t f_bytes = align_up((size_t)C * V * sizeof(float), 256);
    const size_t ws_bytes = align_up(cspn3d_workspace_bytes(1, C, D, H, W, iters), 256);
    const size_t slot_bytes = g_bytes + 2 * f_bytes + ws_bytes;
    int launches = 0;
    for (int b = 0; b < B; ++b) {  // one volume per chunk
        Slot& s = pipe.slots[b % 3];
        int rc = ensure_slot(s, slot_bytes);
        if (rc != CSPN_OK) return rc;
        float* dg = reinterpret_cast<float*>(s.buf);
        float* df = reinterpret_cast<float*>(s.buf + g_bytes);
        float* dout = reinterpret_cast<float*>(s.buf + g_bytes + f_bytes);
        void* dws = ws_bytes ? s.buf + g_bytes + 2 * f_bytes : nullptr;
        CSPN_CUDA_TRY(cudaMemcpyAsync(dg, guidance + (size_t)b * 26 * V, 26 * V * sizeof(float), cudaMemcpyHostToDevice, s.stream));
        CSPN_CUDA_TRY(cudaMemcpyAsync(df, feat + (size_t)b * C * V, (size_t)C * V * sizeof(float), cudaMemcpyHostToDevice, s.stream));
        rc = cspn3d_fwd_f32(dg, df, dout, 1, C, D, H, W, iters, norm_type, dws, ws_bytes, (cspn_stream_t)s.stream);
        if (rc != CSPN_OK) return rc;
        launches += g_last_launches;
        CSPN_CUDA_TRY(cudaMemcpyAsync(out + (size_t)b * C * V, dout, (size_t)C * V * sizeof(float), cudaMemcpyDeviceToHost, s.stream));
    }
    for (auto& s : pipe.slots)
        if (s.stream) CSPN_CUDA_TRY(cudaStreamSynchronize(s.stream));
    drain.armed = false;
    g_last_launches = launches;
    return CSPN_OK;
}
