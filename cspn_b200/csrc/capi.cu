// extern "C" surface of libcspn_b200.so (include/cspn_b200.h): argument checking, algorithm
// dispatch, and the chunked host-buffer pipeline behind the *_host entry points.
#include <cstdlib>
#include <initializer_list>
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

bool kernel_size_ok(int nd, int K) { return K == 3 || K == 5 || (nd == 2 && K == 7); }

template <class... Ints>
bool positive(Ints... v) { return ((v > 0) && ...); }

// The argument check of every propagation entry: nd = 2 (D is 1; K in {3, 5, 7}; norm_type '8sum' / '8sum_abs') or 3 (K in
// {3, 5}; norm_type up to 'paddle').  a, b, c are the entry's three mandatory tensors.  An entry without a kernel size
// passes K = 3, one without a norm_type passes 0, and gch is the 2D guidance's channel count (K*K-1 where the shape implies it).
int check_prop(int nd, const void* a, const void* b, const void* c, int B, int C, int D, int H, int W, int K, int gch, int iters,
               int norm_type) {
    if (!a || !b || !c) { set_error("null tensor pointer"); return CSPN_ERR_INVALID_ARGUMENT; }
    if (!positive(B, C, D, H, W)) {
        if (nd == 2) set_error("non-positive shape B=%d C=%d H=%d W=%d", B, C, H, W);
        else set_error("non-positive shape B=%d C=%d D=%d H=%d W=%d", B, C, D, H, W);
        return CSPN_ERR_INVALID_ARGUMENT;
    }
    if (!kernel_size_ok(nd, K)) { set_error("%dD kernel size must be %s, got %d", nd, nd == 2 ? "3, 5 or 7" : "3 or 5", K); return CSPN_ERR_INVALID_ARGUMENT; }
    if (nd == 2 && gch < K * K - 1) { set_error("a %dx%d kernel needs >= %d guidance channels, got %d", K, K, K * K - 1, gch); return CSPN_ERR_INVALID_ARGUMENT; }
    if (iters < 0) { set_error("prop_time must be >= 0, got %d", iters); return CSPN_ERR_INVALID_ARGUMENT; }
    if (norm_type < 0 || norm_type > (nd == 2 ? (int)CSPN_NORM_8SUM_ABS : (int)CSPN_NORM_PADDLE)) {
        set_error("unknown %snorm_type %d", nd == 2 ? "" : "3D ", norm_type);
        return CSPN_ERR_INVALID_ARGUMENT;
    }
    return CSPN_OK;
}

int check_algo(int algo) {
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

// The destinations of a fused gather as the C ABI takes them
struct Gather {
    float* const* peer_out;
    int n_peer;
    float* multicast_out;
};

void begin_call() {
    clear_error();
    g_last_launches = 0;
}

// What every device entry does once its arguments are checked (the checks come first: they must not need a device):
// select the device that holds `anchor`, the tensor the entry calls `name`, run launch(&launches), publish the count.
template <class Launch>
int on_device_of(const void* anchor, const char* name, Launch&& launch) {
    DeviceGuard guard(device_of(anchor));
    if (!guard.ok) { set_error("cannot select the device of `%s`", name); return CSPN_ERR_CUDA; }
    int launches = 0;
    const int rc = launch(&launches);
    g_last_launches = launches;
    return rc;
}

// A forward entry and its _gather twin: launch(fan, &launches) with fan null for the plain forward (gather null),
// else the checked destinations
template <class Launch>
int run_forward(const void* anchor, const char* name, const Gather* gather, int iters, Launch&& launch) {
    Fan fan{};
    if (gather) {
        const int rc = check_gather(gather->peer_out, gather->n_peer, gather->multicast_out, iters);
        if (rc != CSPN_OK) return rc;
        fan = make_fan(gather->peer_out, gather->n_peer, gather->multicast_out);
    }
    return on_device_of(anchor, name, [&](int* launches) { return launch(gather ? &fan : nullptr, launches); });
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

// The *_workspace_bytes queries return 0 for arguments their entry would reject.  They differ at iters == 0, where the
// entries copy and need nothing: the forward queries and most backward ones answer 0 there, while cspn2d_bwd_workspace_bytes
// and cspn2d_k_bwd_workspace_bytes pass iters == 0 on to the 3x3 backward's own formula.
static size_t workspace2d(int B, int C, int H, int W, int iters, int algo, bool keep) {
    if (!positive(B, C, H, W, iters)) return 0;
    if (algo != CSPN_ALGO_GENERIC) {
        Problem2D p{nullptr, nullptr, nullptr, nullptr, B, C, H, W, 8, iters, 0};
        char why[8];
        if (cluster2d_supported(p, why, sizeof(why))) return cluster2d_workspace_bytes(B, C, H, W, iters);
        if (algo == CSPN_ALGO_CLUSTER) return 0;   // the forward call will report why it is unsupported
    }
    return generic2d_workspace_bytes(B, C, H, W, iters, keep);
}

size_t cspn2d_workspace_bytes(int B, int C, int H, int W, int iters, int algo) { return workspace2d(B, C, H, W, iters, algo, false); }

// The 3x3 forward once its arguments are checked: cspn2d_fwd_f32 (gather null), cspn2d_fwd_gather_f32 and the 3x3 calls of
// the keep-sparse entries (p.keep)
static int fwd2d_3x3(const Problem2D& p, int algo, const Gather* gather, void* workspace, size_t workspace_bytes,
                     cspn_stream_t stream) {
    return on_device_of(p.blur, "blur", [&](int* launches) {
        char why[256] = "";
        if (gather) {
            if (!cluster2d_supported(p, why, sizeof(why), workspace)) {
                set_error("the fused gather runs in the cluster kernel's epilogue, which cannot take this problem: %s", why);
                return (int)CSPN_ERR_UNSUPPORTED;
            }
            g_last_algo = CSPN_ALGO_CLUSTER;
            return cluster2d_forward(p, workspace, workspace_bytes, (cudaStream_t)stream, launches, gather->peer_out, gather->n_peer,
                                     gather->multicast_out);
        }
        const int chosen = (p.iters == 0) ? CSPN_ALGO_GENERIC : resolve_algo(p, algo, why, sizeof(why), workspace);
        if (chosen < 0) { set_error("cluster kernel unsupported for this problem: %s", why); return chosen; }
        g_last_algo = chosen;
        if (chosen == CSPN_ALGO_GENERIC && algo == CSPN_ALGO_AUTO && p.iters > 0) {
            // AUTO sized its workspace for the cluster kernel (cspn2d_workspace_bytes cannot see the pointers); when the
            // problem then has to take the generic path, say so instead of a bare "workspace too small"
            const size_t need = generic2d_workspace_bytes(p.B, p.C, p.H, p.W, p.iters, p.keep);
            if (!workspace || workspace_bytes < need) {
                set_error("CSPN_ALGO_AUTO falls back to the generic path here (%s), which needs %zu workspace bytes (got %zu): "
                          "query %s(..., CSPN_ALGO_GENERIC) or pass 16-byte aligned tensors and workspace",
                          why[0] ? why : "cluster kernel declined", need, workspace ? workspace_bytes : (size_t)0,
                          p.keep ? "cspn2d_keep_workspace_bytes" : "cspn2d_workspace_bytes");
                return (int)CSPN_ERR_WORKSPACE;
            }
        }
        return (chosen == CSPN_ALGO_CLUSTER) ? cluster2d_forward(p, workspace, workspace_bytes, (cudaStream_t)stream, launches)
                                             : generic2d_forward(p, workspace, workspace_bytes, (cudaStream_t)stream, launches);
    });
}

int cspn2d_fwd_f32(const float* guidance, const float* blur, const float* sparse, float* out, int B, int C, int H,
                   int W, int guidance_channels, int iters, int norm_type, int algo, void* workspace,
                   size_t workspace_bytes, cspn_stream_t stream) {
    begin_call();
    int rc = check_prop(2, guidance, blur, out, B, C, 1, H, W, 3, guidance_channels, iters, norm_type);
    if (rc == CSPN_OK) rc = check_algo(algo);
    if (rc != CSPN_OK) return rc;
    const Problem2D p{guidance, blur, sparse, out, B, C, H, W, guidance_channels, iters, norm_type == CSPN_NORM_8SUM_ABS};
    return fwd2d_3x3(p, algo, nullptr, workspace, workspace_bytes, stream);
}

int cspn2d_fwd_gather_f32(const float* guidance, const float* blur, const float* sparse, float* out, float* const* peer_out,
                          int n_peer, float* multicast_out, int B, int C, int H, int W, int guidance_channels, int iters,
                          int norm_type, void* workspace, size_t workspace_bytes, cspn_stream_t stream) {
    begin_call();
    int rc = check_prop(2, guidance, blur, out, B, C, 1, H, W, 3, guidance_channels, iters, norm_type);
    if (rc == CSPN_OK) rc = check_gather(peer_out, n_peer, multicast_out, iters);
    if (rc != CSPN_OK) return rc;
    const Problem2D p{guidance, blur, sparse, out, B, C, H, W, guidance_channels, iters, norm_type == CSPN_NORM_8SUM_ABS};
    const Gather gather{peer_out, n_peer, multicast_out};
    return fwd2d_3x3(p, CSPN_ALGO_CLUSTER, &gather, workspace, workspace_bytes, stream);
}

size_t cspn2d_bwd_workspace_bytes(int B, int C, int H, int W, int iters) {
    if (!positive(B, C, H, W) || iters < 0) return 0;
    return bwd2d_workspace_bytes(B, C, H, W, iters);
}

int cspn2d_bwd_f32(const float* guidance, const float* blur, const float* sparse, const float* grad_out,
                   float* grad_guidance, float* grad_blur, int B, int C, int H, int W, int guidance_channels,
                   int iters, int norm_type, void* workspace, size_t workspace_bytes, cspn_stream_t stream) {
    begin_call();
    const int rc = check_prop(2, guidance, blur, grad_out, B, C, 1, H, W, 3, guidance_channels, iters, norm_type);
    if (rc != CSPN_OK) return rc;
    return on_device_of(blur, "blur", [&](int* launches) {
        Problem2D p{guidance, blur, sparse, nullptr, B, C, H, W, guidance_channels, iters, norm_type == CSPN_NORM_8SUM_ABS};
        return bwd2d(p, grad_out, grad_guidance, grad_blur, workspace, workspace_bytes, (cudaStream_t)stream, launches);
    });
}

// ---- K x K kernels: K = 3 is the operator above, K = 5 / 7 run in cspn2d_wide.cu ----------------------------------
size_t cspn2d_k_workspace_bytes(int B, int C, int H, int W, int K, int iters) {
    if (!positive(B, C, H, W, iters) || !kernel_size_ok(2, K)) return 0;
    if (K == 3) return cspn2d_workspace_bytes(B, C, H, W, iters, CSPN_ALGO_AUTO);
    return widek_workspace_bytes(B, C, H, W, K, iters, Family::Normalised);
}

// gather null: cspn2d_k_fwd_f32
static int fwd2d_k(const float* guidance, const float* blur, const float* sparse, float* out, const Gather* gather, int B, int C,
                   int H, int W, int guidance_channels, int K, int iters, int norm_type, void* workspace, size_t workspace_bytes,
                   cspn_stream_t stream) {
    begin_call();
    const int rc = check_prop(2, guidance, blur, out, B, C, 1, H, W, K, guidance_channels, iters, norm_type);
    if (rc != CSPN_OK) return rc;
    if (K == 3)
        return gather ? cspn2d_fwd_gather_f32(guidance, blur, sparse, out, gather->peer_out, gather->n_peer, gather->multicast_out, B,
                                              C, H, W, guidance_channels, iters, norm_type, workspace, workspace_bytes, stream)
                      : cspn2d_fwd_f32(guidance, blur, sparse, out, B, C, H, W, guidance_channels, iters, norm_type, CSPN_ALGO_AUTO,
                                       workspace, workspace_bytes, stream);
    return run_forward(blur, "blur", gather, iters, [&](const Fan* fan, int* launches) {
        Problem2D p{guidance, blur, sparse, out, B, C, H, W, guidance_channels, iters, norm_type == CSPN_NORM_8SUM_ABS};
        return widek_forward(p, K, Family::Normalised, workspace, workspace_bytes, (cudaStream_t)stream, launches, fan);
    });
}

int cspn2d_k_fwd_f32(const float* guidance, const float* blur, const float* sparse, float* out, int B, int C, int H, int W,
                     int guidance_channels, int K, int iters, int norm_type, void* workspace, size_t workspace_bytes,
                     cspn_stream_t stream) {
    return fwd2d_k(guidance, blur, sparse, out, nullptr, B, C, H, W, guidance_channels, K, iters, norm_type, workspace,
                   workspace_bytes, stream);
}

int cspn2d_k_fwd_gather_f32(const float* guidance, const float* blur, const float* sparse, float* out, float* const* peer_out,
                            int n_peer, float* multicast_out, int B, int C, int H, int W, int guidance_channels, int K,
                            int iters, int norm_type, void* workspace, size_t workspace_bytes, cspn_stream_t stream) {
    const Gather gather{peer_out, n_peer, multicast_out};
    return fwd2d_k(guidance, blur, sparse, out, &gather, B, C, H, W, guidance_channels, K, iters, norm_type, workspace,
                   workspace_bytes, stream);
}

size_t cspn2d_k_bwd_workspace_bytes(int B, int C, int H, int W, int K, int iters) {
    if (!positive(B, C, H, W) || iters < 0 || !kernel_size_ok(2, K)) return 0;
    if (K == 3) return cspn2d_bwd_workspace_bytes(B, C, H, W, iters);
    return widek_bwd_workspace_bytes(B, C, H, W, K, iters, Family::Normalised);
}

int cspn2d_k_bwd_f32(const float* guidance, const float* blur, const float* sparse, const float* grad_out,
                     float* grad_guidance, float* grad_blur, int B, int C, int H, int W, int guidance_channels, int K,
                     int iters, int norm_type, void* workspace, size_t workspace_bytes, cspn_stream_t stream) {
    begin_call();
    const int rc = check_prop(2, guidance, blur, grad_out, B, C, 1, H, W, K, guidance_channels, iters, norm_type);
    if (rc != CSPN_OK) return rc;
    if (K == 3)
        return cspn2d_bwd_f32(guidance, blur, sparse, grad_out, grad_guidance, grad_blur, B, C, H, W, guidance_channels,
                              iters, norm_type, workspace, workspace_bytes, stream);
    return on_device_of(blur, "blur", [&](int* launches) {
        Problem2D p{guidance, blur, sparse, nullptr, B, C, H, W, guidance_channels, iters, norm_type == CSPN_NORM_8SUM_ABS};
        return widek_backward(p, K, Family::Normalised, grad_out, grad_guidance, grad_blur, workspace, workspace_bytes,
                              (cudaStream_t)stream, launches);
    });
}

// ---- 2D keep-sparse mode, K in {3, 5, 7} (DESIGN.md section 4.13): the 3x3 operator above (cluster or generic path) and
// the K x K one (cspn2d_wide.cu) with m = 1[sparse > 0] and the samples themselves as the replacement.  A null sparse is the
// default mode ----------------------------------------------------------------------------------------------------------
size_t cspn2d_keep_workspace_bytes(int B, int C, int H, int W, int K, int iters, int algo) {
    if (!positive(B, C, H, W, iters) || !kernel_size_ok(2, K) || algo < CSPN_ALGO_AUTO || algo > CSPN_ALGO_CLUSTER) return 0;
    if (K == 3) return workspace2d(B, C, H, W, iters, algo, true);
    return widek_workspace_bytes(B, C, H, W, K, iters, Family::Normalised, true);
}

// gather null: cspn2d_keep_fwd_f32
static int fwd2d_keep(const float* guidance, const float* blur, const float* sparse, float* out, const Gather* gather, int B, int C,
                      int H, int W, int guidance_channels, int K, int iters, int norm_type, int algo, void* workspace,
                      size_t workspace_bytes, cspn_stream_t stream) {
    begin_call();
    int rc = check_prop(2, guidance, blur, out, B, C, 1, H, W, K, guidance_channels, iters, norm_type);
    if (rc == CSPN_OK) rc = check_algo(algo);
    if (rc == CSPN_OK && gather) rc = check_gather(gather->peer_out, gather->n_peer, gather->multicast_out, iters);
    if (rc != CSPN_OK) return rc;
    Problem2D p{guidance, blur, sparse, out, B, C, H, W, guidance_channels, iters, norm_type == CSPN_NORM_8SUM_ABS};
    p.keep = sparse != nullptr;
    if (K == 3) return fwd2d_3x3(p, gather ? CSPN_ALGO_CLUSTER : algo, gather, workspace, workspace_bytes, stream);
    return run_forward(blur, "blur", gather, iters, [&](const Fan* fan, int* launches) {
        return widek_forward(p, K, Family::Normalised, workspace, workspace_bytes, (cudaStream_t)stream, launches, fan);
    });
}

int cspn2d_keep_fwd_f32(const float* guidance, const float* blur, const float* sparse, float* out, int B, int C, int H, int W,
                        int guidance_channels, int K, int iters, int norm_type, int algo, void* workspace, size_t workspace_bytes,
                        cspn_stream_t stream) {
    return fwd2d_keep(guidance, blur, sparse, out, nullptr, B, C, H, W, guidance_channels, K, iters, norm_type, algo, workspace,
                      workspace_bytes, stream);
}

int cspn2d_keep_fwd_gather_f32(const float* guidance, const float* blur, const float* sparse, float* out, float* const* peer_out,
                               int n_peer, float* multicast_out, int B, int C, int H, int W, int guidance_channels, int K,
                               int iters, int norm_type, void* workspace, size_t workspace_bytes, cspn_stream_t stream) {
    const Gather gather{peer_out, n_peer, multicast_out};
    return fwd2d_keep(guidance, blur, sparse, out, &gather, B, C, H, W, guidance_channels, K, iters, norm_type, CSPN_ALGO_AUTO,
                      workspace, workspace_bytes, stream);
}

size_t cspn2d_keep_bwd_workspace_bytes(int B, int C, int H, int W, int K, int iters) {
    if (!positive(B, C, H, W) || iters < 0 || !kernel_size_ok(2, K)) return 0;
    if (K == 3) return bwd2d_workspace_bytes(B, C, H, W, iters, true);
    return widek_bwd_workspace_bytes(B, C, H, W, K, iters, Family::Normalised, true);
}

int cspn2d_keep_bwd_f32(const float* guidance, const float* blur, const float* sparse, const float* grad_out,
                        float* grad_guidance, float* grad_blur, float* grad_sparse, int B, int C, int H, int W,
                        int guidance_channels, int K, int iters, int norm_type, void* workspace, size_t workspace_bytes,
                        cspn_stream_t stream) {
    begin_call();
    const int rc = check_prop(2, guidance, blur, grad_out, B, C, 1, H, W, K, guidance_channels, iters, norm_type);
    if (rc != CSPN_OK) return rc;
    return on_device_of(blur, "blur", [&](int* launches) -> int {
        Problem2D p{guidance, blur, sparse, nullptr, B, C, H, W, guidance_channels, iters, norm_type == CSPN_NORM_8SUM_ABS};
        p.keep = sparse != nullptr;
        // no samples, or no step: the output does not depend on sparse
        if (grad_sparse && (!p.keep || iters == 0))
            CSPN_CUDA_TRY(cudaMemsetAsync(grad_sparse, 0, (size_t)B * H * W * sizeof(float), (cudaStream_t)stream));
        if (K == 3)
            return bwd2d(p, grad_out, grad_guidance, grad_blur, workspace, workspace_bytes, (cudaStream_t)stream, launches, grad_sparse);
        return widek_backward(p, K, Family::Normalised, grad_out, grad_guidance, grad_blur, workspace, workspace_bytes,
                              (cudaStream_t)stream, launches, grad_sparse);
    });
}

// ---- 2D 'paddle' (own-location norm) and caller-supplied gates (fluid.layers.affinity_propagate), K in {3, 5, 7}: every
// K in cspn2d_wide.cu.  Both take (gates, feat) with K*K-1 gate channels, so they share their entries' bodies ----------
static size_t own2d_workspace_bytes(Family family, bool bwd, int B, int C, int H, int W, int K, int iters) {
    if (!positive(B, C, H, W, iters) || !kernel_size_ok(2, K)) return 0;
    return bwd ? widek_bwd_workspace_bytes(B, C, H, W, K, iters, family) : widek_workspace_bytes(B, C, H, W, K, iters, family);
}

// gather null: the plain forward
static int own2d_fwd(Family family, const float* gates, const float* feat, float* out, const Gather* gather, int B, int C, int H,
                     int W, int K, int iters, void* workspace, size_t workspace_bytes, cspn_stream_t stream) {
    begin_call();
    const int rc = check_prop(2, gates, feat, out, B, C, 1, H, W, K, K * K - 1, iters, 0);
    if (rc != CSPN_OK) return rc;
    return run_forward(feat, "feat", gather, iters, [&](const Fan* fan, int* launches) {
        Problem2D p{gates, feat, nullptr, out, B, C, H, W, K * K - 1, iters, 0};
        return widek_forward(p, K, family, workspace, workspace_bytes, (cudaStream_t)stream, launches, fan);
    });
}

static int own2d_bwd(Family family, const float* gates, const float* feat, const float* grad_out, float* grad_gates,
                     float* grad_feat, int B, int C, int H, int W, int K, int iters, void* workspace, size_t workspace_bytes,
                     cspn_stream_t stream) {
    begin_call();
    const int rc = check_prop(2, gates, feat, grad_out, B, C, 1, H, W, K, K * K - 1, iters, 0);
    if (rc != CSPN_OK) return rc;
    return on_device_of(feat, "feat", [&](int* launches) {
        Problem2D p{gates, feat, nullptr, nullptr, B, C, H, W, K * K - 1, iters, 0};
        return widek_backward(p, K, family, grad_out, grad_gates, grad_feat, workspace, workspace_bytes, (cudaStream_t)stream,
                              launches);
    });
}

size_t cspn2d_paddle_workspace_bytes(int B, int C, int H, int W, int K, int iters) {
    return own2d_workspace_bytes(Family::Paddle, false, B, C, H, W, K, iters);
}

int cspn2d_paddle_fwd_f32(const float* guidance, const float* feat, float* out, int B, int C, int H, int W, int K, int iters,
                          void* workspace, size_t workspace_bytes, cspn_stream_t stream) {
    return own2d_fwd(Family::Paddle, guidance, feat, out, nullptr, B, C, H, W, K, iters, workspace, workspace_bytes, stream);
}

int cspn2d_paddle_fwd_gather_f32(const float* guidance, const float* feat, float* out, float* const* peer_out, int n_peer,
                                 float* multicast_out, int B, int C, int H, int W, int K, int iters, void* workspace,
                                 size_t workspace_bytes, cspn_stream_t stream) {
    const Gather gather{peer_out, n_peer, multicast_out};
    return own2d_fwd(Family::Paddle, guidance, feat, out, &gather, B, C, H, W, K, iters, workspace, workspace_bytes, stream);
}

size_t cspn2d_paddle_bwd_workspace_bytes(int B, int C, int H, int W, int K, int iters) {
    return own2d_workspace_bytes(Family::Paddle, true, B, C, H, W, K, iters);
}

int cspn2d_paddle_bwd_f32(const float* guidance, const float* feat, const float* grad_out, float* grad_guidance, float* grad_feat,
                          int B, int C, int H, int W, int K, int iters, void* workspace, size_t workspace_bytes,
                          cspn_stream_t stream) {
    return own2d_bwd(Family::Paddle, guidance, feat, grad_out, grad_guidance, grad_feat, B, C, H, W, K, iters, workspace,
                     workspace_bytes, stream);
}

size_t cspn2d_gates_workspace_bytes(int B, int C, int H, int W, int K, int iters) {
    return own2d_workspace_bytes(Family::Gates, false, B, C, H, W, K, iters);
}

int cspn2d_gates_fwd_f32(const float* gates, const float* feat, float* out, int B, int C, int H, int W, int K, int iters,
                         void* workspace, size_t workspace_bytes, cspn_stream_t stream) {
    return own2d_fwd(Family::Gates, gates, feat, out, nullptr, B, C, H, W, K, iters, workspace, workspace_bytes, stream);
}

int cspn2d_gates_fwd_gather_f32(const float* gates, const float* feat, float* out, float* const* peer_out, int n_peer,
                                float* multicast_out, int B, int C, int H, int W, int K, int iters, void* workspace,
                                size_t workspace_bytes, cspn_stream_t stream) {
    const Gather gather{peer_out, n_peer, multicast_out};
    return own2d_fwd(Family::Gates, gates, feat, out, &gather, B, C, H, W, K, iters, workspace, workspace_bytes, stream);
}

size_t cspn2d_gates_bwd_workspace_bytes(int B, int C, int H, int W, int K, int iters) {
    return own2d_workspace_bytes(Family::Gates, true, B, C, H, W, K, iters);
}

int cspn2d_gates_bwd_f32(const float* gates, const float* feat, const float* grad_out, float* grad_gates, float* grad_feat,
                         int B, int C, int H, int W, int K, int iters, void* workspace, size_t workspace_bytes,
                         cspn_stream_t stream) {
    return own2d_bwd(Family::Gates, gates, feat, grad_out, grad_gates, grad_feat, B, C, H, W, K, iters, workspace, workspace_bytes,
                     stream);
}

// ---- 3D: the 3x3x3 operator (cspn3d.cu) -----------------------------------------------------------------------------
size_t cspn3d_workspace_bytes(int B, int C, int D, int H, int W, int iters) {
    if (!positive(B, C, D, H, W, iters)) return 0;
    return generic3d_workspace_bytes(B, C, D, H, W, iters);
}

// gather null: cspn3d_fwd_f32
static int fwd3d(const float* guidance, const float* feat, float* out, const Gather* gather, int B, int C, int D, int H, int W,
                 int iters, int norm_type, void* workspace, size_t workspace_bytes, cspn_stream_t stream) {
    begin_call();
    const int rc = check_prop(3, guidance, feat, out, B, C, D, H, W, 3, 0, iters, norm_type);
    if (rc != CSPN_OK) return rc;
    return run_forward(feat, "feat", gather, iters, [&](const Fan* fan, int* launches) {
        return generic3d_forward(guidance, feat, out, B, C, D, H, W, iters, norm_type, workspace, workspace_bytes,
                                 (cudaStream_t)stream, launches, fan);
    });
}

int cspn3d_fwd_f32(const float* guidance, const float* feat, float* out, int B, int C, int D, int H, int W, int iters,
                   int norm_type, void* workspace, size_t workspace_bytes, cspn_stream_t stream) {
    return fwd3d(guidance, feat, out, nullptr, B, C, D, H, W, iters, norm_type, workspace, workspace_bytes, stream);
}

int cspn3d_fwd_gather_f32(const float* guidance, const float* feat, float* out, float* const* peer_out, int n_peer,
                          float* multicast_out, int B, int C, int D, int H, int W, int iters, int norm_type, void* workspace,
                          size_t workspace_bytes, cspn_stream_t stream) {
    const Gather gather{peer_out, n_peer, multicast_out};
    return fwd3d(guidance, feat, out, &gather, B, C, D, H, W, iters, norm_type, workspace, workspace_bytes, stream);
}

// ---- K x K x K kernels (the K = 3 forward is the 3D operator above, everything else runs in cspn3d_wide.cu, the 3x3x3
// backward included) and caller-supplied gates (K in {3, 5}).  The gates entries have no norm_type and pass 0 ----------
static size_t wide3d_workspace_bytes(Family family, bool bwd, int B, int C, int D, int H, int W, int K, int iters) {
    if (!positive(B, C, D, H, W, iters) || !kernel_size_ok(3, K)) return 0;
    if (K == 3 && family != Family::Gates && !bwd) return cspn3d_workspace_bytes(B, C, D, H, W, iters);
    return bwd ? widek3d_bwd_workspace_bytes(C, D, H, W, K, iters, family) : widek3d_workspace_bytes(B, C, D, H, W, K, iters, family);
}

// gather null: the plain forward
static int wide3d_fwd(Family family, const float* guidance, const float* feat, float* out, const Gather* gather, int B, int C,
                      int D, int H, int W, int K, int iters, int norm_type, void* workspace, size_t workspace_bytes,
                      cspn_stream_t stream) {
    begin_call();
    const int rc = check_prop(3, guidance, feat, out, B, C, D, H, W, K, 0, iters, norm_type);
    if (rc != CSPN_OK) return rc;
    if (K == 3 && family != Family::Gates)
        return fwd3d(guidance, feat, out, gather, B, C, D, H, W, iters, norm_type, workspace, workspace_bytes, stream);
    return run_forward(feat, "feat", gather, iters, [&](const Fan* fan, int* launches) {
        return widek3d_forward(guidance, feat, out, B, C, D, H, W, K, iters, family, norm_type, workspace, workspace_bytes,
                               (cudaStream_t)stream, launches, fan);
    });
}

static int wide3d_bwd(Family family, const float* guidance, const float* feat, const float* grad_out, float* grad_guidance,
                      float* grad_feat, int B, int C, int D, int H, int W, int K, int iters, int norm_type, void* workspace,
                      size_t workspace_bytes, cspn_stream_t stream) {
    begin_call();
    const int rc = check_prop(3, guidance, feat, grad_out, B, C, D, H, W, K, 0, iters, norm_type);
    if (rc != CSPN_OK) return rc;
    return on_device_of(feat, "feat", [&](int* launches) {
        return widek3d_backward(guidance, feat, grad_out, grad_guidance, grad_feat, B, C, D, H, W, K, iters, family, norm_type,
                                workspace, workspace_bytes, (cudaStream_t)stream, launches);
    });
}

size_t cspn3d_k_workspace_bytes(int B, int C, int D, int H, int W, int K, int iters) {
    return wide3d_workspace_bytes(Family::Normalised, false, B, C, D, H, W, K, iters);
}

int cspn3d_k_fwd_f32(const float* guidance, const float* feat, float* out, int B, int C, int D, int H, int W, int K, int iters,
                     int norm_type, void* workspace, size_t workspace_bytes, cspn_stream_t stream) {
    return wide3d_fwd(Family::Normalised, guidance, feat, out, nullptr, B, C, D, H, W, K, iters, norm_type, workspace,
                      workspace_bytes, stream);
}

int cspn3d_k_fwd_gather_f32(const float* guidance, const float* feat, float* out, float* const* peer_out, int n_peer,
                            float* multicast_out, int B, int C, int D, int H, int W, int K, int iters, int norm_type,
                            void* workspace, size_t workspace_bytes, cspn_stream_t stream) {
    const Gather gather{peer_out, n_peer, multicast_out};
    return wide3d_fwd(Family::Normalised, guidance, feat, out, &gather, B, C, D, H, W, K, iters, norm_type, workspace,
                      workspace_bytes, stream);
}

size_t cspn3d_k_bwd_workspace_bytes(int B, int C, int D, int H, int W, int K, int iters) {
    return wide3d_workspace_bytes(Family::Normalised, true, B, C, D, H, W, K, iters);
}

size_t cspn3d_bwd_workspace_bytes(int B, int C, int D, int H, int W, int iters) {
    return wide3d_workspace_bytes(Family::Normalised, true, B, C, D, H, W, 3, iters);
}

int cspn3d_bwd_f32(const float* guidance, const float* feat, const float* grad_out, float* grad_guidance, float* grad_feat,
                   int B, int C, int D, int H, int W, int iters, int norm_type, void* workspace, size_t workspace_bytes,
                   cspn_stream_t stream) {
    return wide3d_bwd(Family::Normalised, guidance, feat, grad_out, grad_guidance, grad_feat, B, C, D, H, W, 3, iters, norm_type,
                      workspace, workspace_bytes, stream);
}

int cspn3d_k_bwd_f32(const float* guidance, const float* feat, const float* grad_out, float* grad_guidance, float* grad_feat,
                     int B, int C, int D, int H, int W, int K, int iters, int norm_type, void* workspace, size_t workspace_bytes,
                     cspn_stream_t stream) {
    return wide3d_bwd(Family::Normalised, guidance, feat, grad_out, grad_guidance, grad_feat, B, C, D, H, W, K, iters, norm_type,
                      workspace, workspace_bytes, stream);
}

size_t cspn3d_gates_workspace_bytes(int B, int C, int D, int H, int W, int K, int iters) {
    return wide3d_workspace_bytes(Family::Gates, false, B, C, D, H, W, K, iters);
}

int cspn3d_gates_fwd_f32(const float* gates, const float* feat, float* out, int B, int C, int D, int H, int W, int K, int iters,
                         void* workspace, size_t workspace_bytes, cspn_stream_t stream) {
    return wide3d_fwd(Family::Gates, gates, feat, out, nullptr, B, C, D, H, W, K, iters, 0, workspace, workspace_bytes, stream);
}

int cspn3d_gates_fwd_gather_f32(const float* gates, const float* feat, float* out, float* const* peer_out, int n_peer,
                                float* multicast_out, int B, int C, int D, int H, int W, int K, int iters, void* workspace,
                                size_t workspace_bytes, cspn_stream_t stream) {
    const Gather gather{peer_out, n_peer, multicast_out};
    return wide3d_fwd(Family::Gates, gates, feat, out, &gather, B, C, D, H, W, K, iters, 0, workspace, workspace_bytes, stream);
}

size_t cspn3d_gates_bwd_workspace_bytes(int B, int C, int D, int H, int W, int K, int iters) {
    return wide3d_workspace_bytes(Family::Gates, true, B, C, D, H, W, K, iters);
}

int cspn3d_gates_bwd_f32(const float* gates, const float* feat, const float* grad_out, float* grad_gates, float* grad_feat,
                         int B, int C, int D, int H, int W, int K, int iters, void* workspace, size_t workspace_bytes,
                         cspn_stream_t stream) {
    return wide3d_bwd(Family::Gates, gates, feat, grad_out, grad_gates, grad_feat, B, C, D, H, W, K, iters, 0, workspace,
                      workspace_bytes, stream);
}

// ---- unpool + crop + 3x3 convolution (the guidance and depth heads) ---------------------------------------------------
static int check_unpool_conv(const void* x, const void* weight, const void* out, int B, int Cin, int h, int w, int Cout, int H,
                             int W) {
    if (!x || !weight || !out) { set_error("null tensor pointer"); return CSPN_ERR_INVALID_ARGUMENT; }
    if (!positive(B, Cin, h, w, Cout, H, W)) {
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
    begin_call();
    const int rc = check_unpool_conv(x, weight, out, B, Cin, h, w, Cout, H, W);
    if (rc != CSPN_OK) return rc;
    return on_device_of(x, "x", [&](int* launches) {
        return unpool_conv_forward(x, weight, out, B, Cin, h, w, Cout, H, W, (cudaStream_t)stream, launches);
    });
}

size_t cspn_unpool_conv3x3_bwd_workspace_bytes(int B, int Cin, int h, int w, int Cout, int H, int W) {
    if (!positive(B, Cin, h, w, Cout, H, W) || H > 2 * h || W > 2 * w) return 0;
    return unpool_conv_bwd_workspace_bytes(B, Cin, H, W, Cout);
}

int cspn_unpool_conv3x3_bwd_f32(const float* x, const float* weight, const float* grad_out, float* grad_x, float* grad_weight,
                                int B, int Cin, int h, int w, int Cout, int H, int W, void* workspace, size_t workspace_bytes,
                                cspn_stream_t stream) {
    begin_call();
    const int rc = check_unpool_conv(x, weight, grad_out, B, Cin, h, w, Cout, H, W);
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
    return on_device_of(x, "x", [&](int* launches) {
        return unpool_conv_backward(x, weight, grad_out, grad_x, grad_weight, B, Cin, h, w, Cout, H, W, workspace,
                                    (cudaStream_t)stream, launches);
    });
}

// ---- trilinear resampling (the Paddle module's resize_trilinear) --------------------------------------------------------
// Bytes of a (B*C) x n fp32 tensor, saturated at the top of the address space
static uintptr_t span_bytes(int B, int C, long long n) {
    const unsigned long long lim = ~0ull / 4 / (unsigned long long)n;
    const unsigned long long bc = (unsigned long long)B * C;
    return bc > lim ? ~(uintptr_t)0 : (uintptr_t)(bc * n * 4);
}

static bool overlap(const void* a, uintptr_t na, const void* b, uintptr_t nb) {
    const uintptr_t pa = reinterpret_cast<uintptr_t>(a), pb = reinterpret_cast<uintptr_t>(b);
    const uintptr_t ea = na > ~pa ? ~(uintptr_t)0 : pa + na, eb = nb > ~pb ? ~(uintptr_t)0 : pb + nb;
    return pa < eb && pb < ea;
}

// The sizes, flags and pointers of a resampling entry: src is read and dst written
static int check_resize_args(const void* src, const void* dst, int B, int C, int D, int H, int W, int Do, int Ho, int Wo,
                             int align_corners, int align_mode) {
    if (!src || !dst) { set_error("null tensor pointer"); return CSPN_ERR_INVALID_ARGUMENT; }
    if (!positive(B, C, D, H, W, Do, Ho, Wo)) {
        set_error("non-positive size B=%d C=%d D=%d H=%d W=%d Do=%d Ho=%d Wo=%d", B, C, D, H, W, Do, Ho, Wo);
        return CSPN_ERR_INVALID_ARGUMENT;
    }
    if (align_corners != 0 && align_corners != 1) { set_error("align_corners must be 0 or 1, got %d", align_corners); return CSPN_ERR_INVALID_ARGUMENT; }
    if (align_mode != 0 && align_mode != 1) { set_error("align_mode must be 0 or 1, got %d", align_mode); return CSPN_ERR_INVALID_ARGUMENT; }
    if ((reinterpret_cast<uintptr_t>(src) | reinterpret_cast<uintptr_t>(dst)) & 3) {
        set_error("tensor pointers must be 4-byte aligned");
        return CSPN_ERR_INVALID_ARGUMENT;
    }
    const char* why = "";
    if (!resize_trilinear_launchable(D, H, W, Do, Ho, Wo, &why)) { set_error("unsupported shape: %s", why); return CSPN_ERR_UNSUPPORTED; }
    return CSPN_OK;
}

// src is read and dst written: x and out in the forward, grad_out and grad_x in the backward
static int check_resize(const void* src, const void* dst, int B, int C, int D, int H, int W, int Do, int Ho, int Wo,
                        int align_corners, int align_mode, bool backward) {
    const int rc = check_resize_args(src, dst, B, C, D, H, W, Do, Ho, Wo, align_corners, align_mode);
    if (rc != CSPN_OK) return rc;
    const long long vin = (long long)D * H * W, vout = (long long)Do * Ho * Wo;
    if (overlap(src, span_bytes(B, C, backward ? vout : vin), dst, span_bytes(B, C, backward ? vin : vout))) {
        set_error("%s overlaps %s", backward ? "grad_x" : "out", backward ? "grad_out" : "x");
        return CSPN_ERR_INVALID_ARGUMENT;
    }
    return CSPN_OK;
}

int cspn_resize_trilinear_fwd_f32(const float* x, float* out, int B, int C, int D, int H, int W, int Do, int Ho, int Wo,
                                  int align_corners, int align_mode, cspn_stream_t stream) {
    begin_call();
    const int rc = check_resize(x, out, B, C, D, H, W, Do, Ho, Wo, align_corners, align_mode, false);
    if (rc != CSPN_OK) return rc;
    return on_device_of(x, "x", [&](int* launches) {
        return resize_trilinear_forward(x, out, (long long)B * C, D, H, W, Do, Ho, Wo, align_corners, align_mode,
                                        (cudaStream_t)stream, launches);
    });
}

size_t cspn_resize_trilinear_bwd_workspace_bytes(int D, int H, int W, int Do, int Ho, int Wo) {
    if (!positive(D, H, W, Do, Ho, Wo)) return 0;
    return resize_trilinear_bwd_workspace_bytes(D, H, W, Do, Ho, Wo);
}

int cspn_resize_trilinear_bwd_f32(const float* grad_out, float* grad_x, int B, int C, int D, int H, int W, int Do, int Ho,
                                  int Wo, int align_corners, int align_mode, void* workspace, size_t workspace_bytes,
                                  cspn_stream_t stream) {
    begin_call();
    const int rc = check_resize(grad_out, grad_x, B, C, D, H, W, Do, Ho, Wo, align_corners, align_mode, true);
    if (rc != CSPN_OK) return rc;
    const size_t need = resize_trilinear_bwd_workspace_bytes(D, H, W, Do, Ho, Wo);
    if (!workspace || workspace_bytes < need || (reinterpret_cast<uintptr_t>(workspace) & 7)) {
        set_error("the backward needs %zu bytes of 8-byte aligned workspace (got %zu)", need, workspace_bytes);
        return CSPN_ERR_WORKSPACE;
    }
    const long long vin = (long long)D * H * W, vout = (long long)Do * Ho * Wo;
    if (overlap(workspace, need, grad_x, span_bytes(B, C, vin)) || overlap(workspace, need, grad_out, span_bytes(B, C, vout))) {
        set_error("the workspace overlaps %s", overlap(workspace, need, grad_x, span_bytes(B, C, vin)) ? "grad_x" : "grad_out");
        return CSPN_ERR_INVALID_ARGUMENT;
    }
    return on_device_of(grad_out, "grad_out", [&](int* launches) {
        return resize_trilinear_backward(grad_out, grad_x, (long long)B * C, D, H, W, Do, Ho, Wo, align_corners, align_mode,
                                         workspace, (cudaStream_t)stream, launches);
    });
}

// ---- disparity regression from a low-resolution cost volume (resize_trilinear, softmax over d, expectation) ---------------
// resize's argument check, then the tile rule: cost is read and dst (out, or grad_cost) written
static int check_disparity(const float* cost, const float* dst, int B, int C, int D, int H, int W, int Do, int Ho, int Wo,
                           int align_corners, int align_mode) {
    int rc = check_resize_args(cost, dst, B, C, D, H, W, Do, Ho, Wo, align_corners, align_mode);
    if (rc != CSPN_OK) return rc;
    const char* why = "";
    if (!disparity_regression_launchable(D, H, W, Do, Ho, Wo, align_corners, align_mode, &why)) {
        set_error("unsupported shape: %s", why);
        return CSPN_ERR_UNSUPPORTED;
    }
    return CSPN_OK;
}

int cspn_disparity_regression_fwd_f32(const float* cost, float* out, int B, int C, int D, int H, int W, int Do, int Ho, int Wo,
                                      int align_corners, int align_mode, cspn_stream_t stream) {
    begin_call();
    const int rc = check_disparity(cost, out, B, C, D, H, W, Do, Ho, Wo, align_corners, align_mode);
    if (rc != CSPN_OK) return rc;
    if (overlap(cost, span_bytes(B, C, (long long)D * H * W), out, span_bytes(B, C, (long long)Ho * Wo))) {
        set_error("out overlaps cost");
        return CSPN_ERR_INVALID_ARGUMENT;
    }
    return on_device_of(cost, "cost", [&](int* launches) {
        return disparity_regression_forward(cost, out, (long long)B * C, D, H, W, Do, Ho, Wo, align_corners, align_mode,
                                            (cudaStream_t)stream, launches);
    });
}

size_t cspn_disparity_regression_bwd_workspace_bytes(int D, int H, int W, int Do, int Ho, int Wo) {
    return cspn_resize_trilinear_bwd_workspace_bytes(D, H, W, Do, Ho, Wo);
}

int cspn_disparity_regression_bwd_f32(const float* cost, const float* grad_out, float* grad_cost, int B, int C, int D, int H,
                                      int W, int Do, int Ho, int Wo, int align_corners, int align_mode, void* workspace,
                                      size_t workspace_bytes, cspn_stream_t stream) {
    begin_call();
    const int rc = check_disparity(cost, grad_cost, B, C, D, H, W, Do, Ho, Wo, align_corners, align_mode);
    if (rc != CSPN_OK) return rc;
    if (!grad_out) { set_error("null tensor pointer"); return CSPN_ERR_INVALID_ARGUMENT; }
    if (reinterpret_cast<uintptr_t>(grad_out) & 3) { set_error("tensor pointers must be 4-byte aligned"); return CSPN_ERR_INVALID_ARGUMENT; }
    const uintptr_t n_cost = span_bytes(B, C, (long long)D * H * W), n_g = span_bytes(B, C, (long long)Ho * Wo);
    if (overlap(grad_cost, n_cost, cost, n_cost) || overlap(grad_cost, n_cost, grad_out, n_g)) {
        set_error("grad_cost overlaps %s", overlap(grad_cost, n_cost, cost, n_cost) ? "cost" : "grad_out");
        return CSPN_ERR_INVALID_ARGUMENT;
    }
    const size_t need = resize_trilinear_bwd_workspace_bytes(D, H, W, Do, Ho, Wo);
    if (!workspace || workspace_bytes < need || (reinterpret_cast<uintptr_t>(workspace) & 7)) {
        set_error("the backward needs %zu bytes of 8-byte aligned workspace (got %zu)", need, workspace_bytes);
        return CSPN_ERR_WORKSPACE;
    }
    const char* hit = overlap(workspace, need, grad_cost, n_cost) ? "grad_cost"
                      : overlap(workspace, need, cost, n_cost)    ? "cost"
                      : overlap(workspace, need, grad_out, n_g)   ? "grad_out"
                                                                  : nullptr;
    if (hit) { set_error("the workspace overlaps %s", hit); return CSPN_ERR_INVALID_ARGUMENT; }
    return on_device_of(cost, "cost", [&](int* launches) {
        return disparity_regression_backward(cost, grad_out, grad_cost, (long long)B * C, D, H, W, Do, Ho, Wo, align_corners,
                                             align_mode, workspace, (cudaStream_t)stream, launches);
    });
}

// ---- stereo cost volumes (concatenation and group-wise correlation) -------------------------------------------------------
// The sizes and F % G of an entry (G == 0: the concatenation volume); checked before any byte count is formed
static int check_cost_volume_sizes(int B, int F, int H, int W, int D, int G, bool gwc) {
    if (!positive(B, F, H, W, D) || (gwc && G < 1)) {
        set_error("non-positive size B=%d F=%d H=%d W=%d D=%d%s", B, F, H, W, D, gwc && G < 1 ? " or G < 1" : "");
        return CSPN_ERR_INVALID_ARGUMENT;
    }
    if (gwc && F % G != 0) { set_error("num_groups=%d must divide F=%d", G, F); return CSPN_ERR_INVALID_ARGUMENT; }
    return CSPN_OK;
}

struct Buf {
    const void* p;
    uintptr_t bytes;
    const char* name;
};

// The pointers of an entry, the tile rule, then the overlaps: `in` are read and `outs` written.  An output may overlap neither an input
// nor another output; inputs may alias one another (left may be right).
static int check_cost_volume(int F, int H, int W, int D, int G, std::initializer_list<Buf> in, std::initializer_list<Buf> outs) {
    uintptr_t bits = 0;
    for (const auto* set : {&in, &outs})
        for (const Buf& b : *set) {
            if (!b.p) { set_error("null tensor pointer"); return CSPN_ERR_INVALID_ARGUMENT; }
            bits |= reinterpret_cast<uintptr_t>(b.p);
        }
    if (bits & 3) { set_error("tensor pointers must be 4-byte aligned"); return CSPN_ERR_INVALID_ARGUMENT; }
    if (2ll * F >= (1ll << 31)) { set_error("unsupported shape: 2F >= 2^31 channels"); return CSPN_ERR_UNSUPPORTED; }
    const char* why = "";
    if (!cost_volume_launchable(F, H, W, D, G, &why)) { set_error("unsupported shape: %s", why); return CSPN_ERR_UNSUPPORTED; }
    for (const Buf& o : outs) {
        for (const Buf& i : in)
            if (overlap(o.p, o.bytes, i.p, i.bytes)) { set_error("%s overlaps %s", o.name, i.name); return CSPN_ERR_INVALID_ARGUMENT; }
        for (const Buf& o2 : outs)
            if (&o2 < &o && overlap(o.p, o.bytes, o2.p, o2.bytes)) {
                set_error("%s overlaps %s", o.name, o2.name);
                return CSPN_ERR_INVALID_ARGUMENT;
            }
    }
    return CSPN_OK;
}

int cspn_concat_volume_fwd_f32(const float* left, const float* right, float* out, int B, int F, int H, int W, int D,
                               cspn_stream_t stream) {
    begin_call();
    int rc = check_cost_volume_sizes(B, F, H, W, D, 0, false);
    if (rc != CSPN_OK) return rc;
    const uintptr_t n_in = span_bytes(B, F, (long long)H * W), n_out = span_bytes(B, F, 2ll * D * H * W);
    rc = check_cost_volume(F, H, W, D, 0, {{left, n_in, "left"}, {right, n_in, "right"}}, {{out, n_out, "out"}});
    if (rc != CSPN_OK) return rc;
    return on_device_of(left, "left", [&](int* launches) {
        return concat_volume_forward(left, right, out, B, F, H, W, D, (cudaStream_t)stream, launches);
    });
}

int cspn_concat_volume_bwd_f32(const float* grad_out, float* grad_left, float* grad_right, int B, int F, int H, int W, int D,
                               cspn_stream_t stream) {
    begin_call();
    int rc = check_cost_volume_sizes(B, F, H, W, D, 0, false);
    if (rc != CSPN_OK) return rc;
    const uintptr_t n_in = span_bytes(B, F, (long long)H * W), n_g = span_bytes(B, F, 2ll * D * H * W);
    rc = check_cost_volume(F, H, W, D, 0, {{grad_out, n_g, "grad_out"}},
                           {{grad_left, n_in, "grad_left"}, {grad_right, n_in, "grad_right"}});
    if (rc != CSPN_OK) return rc;
    return on_device_of(grad_out, "grad_out", [&](int* launches) {
        return concat_volume_backward(grad_out, grad_left, grad_right, B, F, H, W, D, (cudaStream_t)stream, launches);
    });
}

int cspn_gwc_volume_fwd_f32(const float* left, const float* right, float* out, int B, int F, int H, int W, int D, int G,
                            cspn_stream_t stream) {
    begin_call();
    int rc = check_cost_volume_sizes(B, F, H, W, D, G, true);
    if (rc != CSPN_OK) return rc;
    const uintptr_t n_in = span_bytes(B, F, (long long)H * W), n_out = span_bytes(B, G, (long long)D * H * W);
    rc = check_cost_volume(F, H, W, D, G, {{left, n_in, "left"}, {right, n_in, "right"}}, {{out, n_out, "out"}});
    if (rc != CSPN_OK) return rc;
    return on_device_of(left, "left", [&](int* launches) {
        return gwc_volume_forward(left, right, out, B, F, H, W, D, G, (cudaStream_t)stream, launches);
    });
}

int cspn_gwc_volume_bwd_f32(const float* left, const float* right, const float* grad_out, float* grad_left, float* grad_right,
                            int B, int F, int H, int W, int D, int G, cspn_stream_t stream) {
    begin_call();
    int rc = check_cost_volume_sizes(B, F, H, W, D, G, true);
    if (rc != CSPN_OK) return rc;
    const uintptr_t n_in = span_bytes(B, F, (long long)H * W), n_g = span_bytes(B, G, (long long)D * H * W);
    rc = check_cost_volume(F, H, W, D, G, {{left, n_in, "left"}, {right, n_in, "right"}, {grad_out, n_g, "grad_out"}},
                           {{grad_left, n_in, "grad_left"}, {grad_right, n_in, "grad_right"}});
    if (rc != CSPN_OK) return rc;
    return on_device_of(left, "left", [&](int* launches) {
        return gwc_volume_backward(left, right, grad_out, grad_left, grad_right, B, F, H, W, D, G, (cudaStream_t)stream,
                                   launches);
    });
}

// ---- affinity pooling (the CSPN stereo network's spatial pyramid pooling) ---------------------------------------------------
// The sizes, the levels, the pointers, the launch limits, then the overlaps, in that order: `in` are read and `outs` written.
// *n_out is the packed output's element count per (B, channel), sum_l (H / p_l) * (W / p_l).
static int check_affinity_pool(int B, int C, int H, int W, int L, const int* ks, long long* n_out,
                               std::initializer_list<Buf> in, std::initializer_list<Buf> outs) {
    if (!positive(B, C, H, W)) { set_error("non-positive size B=%d C=%d H=%d W=%d", B, C, H, W); return CSPN_ERR_INVALID_ARGUMENT; }
    if (L < 1 || L > kAffinityPoolMaxLevels) { set_error("the number of levels L=%d must be 1..8", L); return CSPN_ERR_INVALID_ARGUMENT; }
    if (!ks) { set_error("null kernel_sizes"); return CSPN_ERR_INVALID_ARGUMENT; }
    const int lim = H < W ? H : W;
    *n_out = 0;
    for (int l = 0; l < L; ++l) {
        if (ks[l] < 1 || ks[l] > lim) {
            set_error("kernel_sizes[%d]=%d must be in [1, min(H, W)=%d]", l, ks[l], lim);
            return CSPN_ERR_INVALID_ARGUMENT;
        }
        *n_out += (long long)(H / ks[l]) * (W / ks[l]);
    }
    uintptr_t bits = 0;
    for (const auto* set : {&in, &outs})
        for (const Buf& b : *set) {
            if (!b.p) { set_error("null tensor pointer"); return CSPN_ERR_INVALID_ARGUMENT; }
            bits |= reinterpret_cast<uintptr_t>(b.p);
        }
    if (bits & 3) { set_error("tensor pointers must be 4-byte aligned"); return CSPN_ERR_INVALID_ARGUMENT; }
    const char* why = "";
    if (!affinity_pool_launchable(B, C, H, W, L, ks, &why)) { set_error("unsupported shape: %s", why); return CSPN_ERR_UNSUPPORTED; }
    return CSPN_OK;
}

// An output may overlap neither an input nor another output; inputs may alias one another
static int check_disjoint(const std::vector<Buf>& in, const std::vector<Buf>& outs) {
    for (const Buf& o : outs) {
        for (const Buf& i : in)
            if (overlap(o.p, o.bytes, i.p, i.bytes)) { set_error("%s overlaps %s", o.name, i.name); return CSPN_ERR_INVALID_ARGUMENT; }
        for (const Buf& o2 : outs)
            if (&o2 < &o && overlap(o.p, o.bytes, o2.p, o2.bytes)) {
                set_error("%s overlaps %s", o.name, o2.name);
                return CSPN_ERR_INVALID_ARGUMENT;
            }
    }
    return CSPN_OK;
}

int cspn_affinity_pool2d_fwd_f32(const float* feat, const float* gate, float* out, int B, int C, int H, int W, int L,
                                 const int* kernel_sizes, cspn_stream_t stream) {
    begin_call();
    long long n;
    int rc = check_affinity_pool(B, C, H, W, L, kernel_sizes, &n, {{feat, 0, "feat"}, {gate, 0, "gate"}}, {{out, 0, "out"}});
    if (rc != CSPN_OK) return rc;
    rc = check_disjoint({{feat, span_bytes(B, C, (long long)H * W), "feat"}, {gate, span_bytes(B, L, (long long)H * W), "gate"}},
                        {{out, span_bytes(B, C, n), "out"}});
    if (rc != CSPN_OK) return rc;
    return on_device_of(feat, "feat", [&](int* launches) {
        return affinity_pool_forward(feat, gate, out, B, C, H, W, L, kernel_sizes, (cudaStream_t)stream, launches);
    });
}

int cspn_affinity_pool2d_bwd_f32(const float* feat, const float* gate, const float* out, const float* grad_out,
                                 float* grad_feat, float* grad_gate, int B, int C, int H, int W, int L, const int* kernel_sizes,
                                 cspn_stream_t stream) {
    begin_call();
    long long n;
    int rc = check_affinity_pool(B, C, H, W, L, kernel_sizes, &n,
                                 {{feat, 0, "feat"}, {gate, 0, "gate"}, {out, 0, "out"}, {grad_out, 0, "grad_out"}},
                                 {{grad_feat, 0, "grad_feat"}, {grad_gate, 0, "grad_gate"}});
    if (rc != CSPN_OK) return rc;
    const uintptr_t n_f = span_bytes(B, C, (long long)H * W), n_g = span_bytes(B, L, (long long)H * W), n_o = span_bytes(B, C, n);
    rc = check_disjoint({{feat, n_f, "feat"}, {gate, n_g, "gate"}, {out, n_o, "out"}, {grad_out, n_o, "grad_out"}},
                        {{grad_feat, n_f, "grad_feat"}, {grad_gate, n_g, "grad_gate"}});
    if (rc != CSPN_OK) return rc;
    return on_device_of(feat, "feat", [&](int* launches) {
        return affinity_pool_backward(feat, gate, out, grad_out, grad_feat, grad_gate, B, C, H, W, L, kernel_sizes,
                                      (cudaStream_t)stream, launches);
    });
}

// ---- affinity fusion (the CSPN stereo network's spatial pyramid fusion) ----------------------------------------------------
// The sizes, the levels, the flags, the pointers, then the launch limits: `in` are read and `outs` written, and the level
// pointers join them (grad_levels only in the backward).  On success n_lvl[l] is level l's elements per (B, channel).
static int check_affinity_fuse(int B, int C, int H, int W, int L, const int* level_hw, int align_corners, int align_mode,
                               const float* const* levels, float* const* grad_levels, bool backward, long long* n_lvl,
                               std::vector<Buf> in, std::vector<Buf> outs) {
    if (!positive(B, C, H, W)) { set_error("non-positive size B=%d C=%d H=%d W=%d", B, C, H, W); return CSPN_ERR_INVALID_ARGUMENT; }
    if (L < 1 || L > kAffinityFuseMaxLevels) { set_error("the number of levels L=%d must be 1..8", L); return CSPN_ERR_INVALID_ARGUMENT; }
    if (!level_hw) { set_error("null level_hw"); return CSPN_ERR_INVALID_ARGUMENT; }
    for (int l = 0; l < L; ++l) {
        if (!positive(level_hw[2 * l], level_hw[2 * l + 1])) {
            set_error("non-positive size %dx%d of level %d", level_hw[2 * l], level_hw[2 * l + 1], l);
            return CSPN_ERR_INVALID_ARGUMENT;
        }
        n_lvl[l] = (long long)level_hw[2 * l] * level_hw[2 * l + 1];
    }
    if (align_corners != 0 && align_corners != 1) { set_error("align_corners must be 0 or 1, got %d", align_corners); return CSPN_ERR_INVALID_ARGUMENT; }
    if (align_mode != 0 && align_mode != 1) { set_error("align_mode must be 0 or 1, got %d", align_mode); return CSPN_ERR_INVALID_ARGUMENT; }
    if (!levels || (backward && !grad_levels)) { set_error("null level pointer array"); return CSPN_ERR_INVALID_ARGUMENT; }
    for (int l = 0; l < L; ++l) {
        in.push_back({levels[l], 0, "levels[]"});
        if (backward) outs.push_back({grad_levels[l], 0, "grad_levels[]"});
    }
    uintptr_t bits = 0;
    for (const auto* set : {&in, &outs})
        for (const Buf& b : *set) {
            if (!b.p) { set_error("null tensor pointer"); return CSPN_ERR_INVALID_ARGUMENT; }
            bits |= reinterpret_cast<uintptr_t>(b.p);
        }
    if (bits & 3) { set_error("tensor pointers must be 4-byte aligned"); return CSPN_ERR_INVALID_ARGUMENT; }
    const char* why = "";
    if (!affinity_fuse_launchable(B, C, H, W, L, level_hw, &why)) { set_error("unsupported shape: %s", why); return CSPN_ERR_UNSUPPORTED; }
    return CSPN_OK;
}

// The level buffers as overlap operands, named levels[l] or grad_levels[l]
using LevelNames = char[kAffinityFuseMaxLevels][24];
static void add_levels(std::vector<Buf>& set, const float* const* p, int B, int C, int L, const long long* n_lvl, const char* what,
                       LevelNames& names) {
    for (int l = 0; l < L; ++l) {
        snprintf(names[l], sizeof(names[l]), "%s[%d]", what, l);
        set.push_back({p[l], span_bytes(B, C, n_lvl[l]), names[l]});
    }
}

int cspn_affinity_fuse2d_fwd_f32(const float* const* levels, const int* level_hw, const float* gate, float* out, int B, int C,
                                 int H, int W, int L, int align_corners, int align_mode, cspn_stream_t stream) {
    begin_call();
    long long n_lvl[kAffinityFuseMaxLevels];
    int rc = check_affinity_fuse(B, C, H, W, L, level_hw, align_corners, align_mode, levels, nullptr, false, n_lvl,
                                 {{gate, 0, "gate"}}, {{out, 0, "out"}});
    if (rc != CSPN_OK) return rc;
    LevelNames names;
    std::vector<Buf> in{{gate, span_bytes(B, L, (long long)H * W), "gate"}};
    add_levels(in, levels, B, C, L, n_lvl, "levels", names);
    rc = check_disjoint(in, {{out, span_bytes(B, C, (long long)H * W), "out"}});
    if (rc != CSPN_OK) return rc;
    return on_device_of(gate, "gate", [&](int* launches) {
        return affinity_fuse_forward(levels, level_hw, gate, out, B, C, H, W, L, align_corners, align_mode, (cudaStream_t)stream,
                                     launches);
    });
}

size_t cspn_affinity_fuse2d_bwd_workspace_bytes(int B, int C, int H, int W, int L, const int* level_hw) {
    if (!positive(B, C, H, W) || L < 1 || L > kAffinityFuseMaxLevels || !level_hw) return 0;
    for (int l = 0; l < 2 * L; ++l)
        if (level_hw[l] < 1) return 0;
    return affinity_fuse_bwd_workspace_bytes(B, C, H, W, L, level_hw);
}

int cspn_affinity_fuse2d_bwd_f32(const float* const* levels, const int* level_hw, const float* gate, const float* out,
                                 const float* grad_out, float* const* grad_levels, float* grad_gate, int B, int C, int H, int W,
                                 int L, int align_corners, int align_mode, void* workspace, size_t workspace_bytes,
                                 cspn_stream_t stream) {
    begin_call();
    long long n_lvl[kAffinityFuseMaxLevels];
    int rc = check_affinity_fuse(B, C, H, W, L, level_hw, align_corners, align_mode, levels, grad_levels, true, n_lvl,
                                 {{gate, 0, "gate"}, {out, 0, "out"}, {grad_out, 0, "grad_out"}}, {{grad_gate, 0, "grad_gate"}});
    if (rc != CSPN_OK) return rc;
    const size_t need = affinity_fuse_bwd_workspace_bytes(B, C, H, W, L, level_hw);
    if (!workspace || workspace_bytes < need || (reinterpret_cast<uintptr_t>(workspace) & 3)) {
        set_error("the backward needs %zu bytes of 4-byte aligned workspace (got %zu)", need, workspace_bytes);
        return CSPN_ERR_WORKSPACE;
    }
    const uintptr_t n_g = span_bytes(B, L, (long long)H * W), n_o = span_bytes(B, C, (long long)H * W);
    LevelNames in_names, out_names;
    std::vector<Buf> in{{gate, n_g, "gate"}, {out, n_o, "out"}, {grad_out, n_o, "grad_out"}};
    std::vector<Buf> outs{{grad_gate, n_g, "grad_gate"}, {workspace, need, "the workspace"}};
    add_levels(in, levels, B, C, L, n_lvl, "levels", in_names);
    add_levels(outs, grad_levels, B, C, L, n_lvl, "grad_levels", out_names);
    rc = check_disjoint(in, outs);
    if (rc != CSPN_OK) return rc;
    return on_device_of(gate, "gate", [&](int* launches) {
        return affinity_fuse_backward(levels, level_hw, gate, out, grad_out, grad_levels, grad_gate, B, C, H, W, L, align_corners,
                                      align_mode, workspace, (cudaStream_t)stream, launches);
    });
}

// ---- atrous affinity pooling (the CSPN stereo network's ACSPP) ---------------------------------------------------------------
// The sizes, the levels and the rates: true when they are valid (the error is set otherwise)
static bool atrous_args_ok(int B, int C, int H, int W, int L, const int* dilations) {
    if (!positive(B, C, H, W)) { set_error("non-positive size B=%d C=%d H=%d W=%d", B, C, H, W); return false; }
    if (L < 1 || L > kAffinityAtrousMaxLevels) { set_error("the number of levels L=%d must be 1..8", L); return false; }
    if (!dilations) { set_error("null dilations"); return false; }
    const int lim = H > W ? H : W;
    for (int l = 0; l < L; ++l)
        if (dilations[l] < 1 || dilations[l] > lim) {
            set_error("dilations[%d]=%d must be in [1, max(H, W)=%d]", l, dilations[l], lim);
            return false;
        }
    return true;
}

// The sizes, the rates, the pointers, then the launch limits: `in` are read and `outs` written
static int check_affinity_atrous(int B, int C, int H, int W, int L, const int* dilations, std::initializer_list<Buf> in,
                                 std::initializer_list<Buf> outs) {
    if (!atrous_args_ok(B, C, H, W, L, dilations)) return CSPN_ERR_INVALID_ARGUMENT;
    uintptr_t bits = 0;
    for (const auto* set : {&in, &outs})
        for (const Buf& b : *set) {
            if (!b.p) { set_error("null tensor pointer"); return CSPN_ERR_INVALID_ARGUMENT; }
            bits |= reinterpret_cast<uintptr_t>(b.p);
        }
    if (bits & 3) { set_error("tensor pointers must be 4-byte aligned"); return CSPN_ERR_INVALID_ARGUMENT; }
    const char* why = "";
    if (!affinity_atrous_launchable(B, C, H, W, L, &why)) { set_error("unsupported shape: %s", why); return CSPN_ERR_UNSUPPORTED; }
    return CSPN_OK;
}

int cspn_affinity_atrous2d_fwd_f32(const float* feat, const float* gate, float* out, int B, int C, int H, int W, int L,
                                   const int* dilations, cspn_stream_t stream) {
    begin_call();
    int rc = check_affinity_atrous(B, C, H, W, L, dilations, {{feat, 0, "feat"}, {gate, 0, "gate"}}, {{out, 0, "out"}});
    if (rc != CSPN_OK) return rc;
    const long long hw = (long long)H * W;
    rc = check_disjoint({{feat, span_bytes(B, C, hw), "feat"}, {gate, span_bytes(B, 9 * L, hw), "gate"}},
                        {{out, span_bytes(B, C, L * hw), "out"}});
    if (rc != CSPN_OK) return rc;
    return on_device_of(feat, "feat", [&](int* launches) {
        return affinity_atrous_forward(feat, gate, out, B, C, H, W, L, dilations, (cudaStream_t)stream, launches);
    });
}

size_t cspn_affinity_atrous2d_bwd_workspace_bytes(int B, int C, int H, int W, int L, const int* dilations) {
    if (!atrous_args_ok(B, C, H, W, L, dilations)) return 0;
    return affinity_atrous_bwd_workspace_bytes(B, H, W, L);
}

int cspn_affinity_atrous2d_bwd_f32(const float* feat, const float* gate, const float* out, const float* grad_out,
                                   float* grad_feat, float* grad_gate, int B, int C, int H, int W, int L, const int* dilations,
                                   void* workspace, size_t workspace_bytes, cspn_stream_t stream) {
    begin_call();
    int rc = check_affinity_atrous(B, C, H, W, L, dilations,
                                   {{feat, 0, "feat"}, {gate, 0, "gate"}, {out, 0, "out"}, {grad_out, 0, "grad_out"}},
                                   {{grad_feat, 0, "grad_feat"}, {grad_gate, 0, "grad_gate"}});
    if (rc != CSPN_OK) return rc;
    const size_t need = affinity_atrous_bwd_workspace_bytes(B, H, W, L);
    if (!workspace || workspace_bytes < need || (reinterpret_cast<uintptr_t>(workspace) & 3)) {
        set_error("the backward needs %zu bytes of 4-byte aligned workspace (got %zu)", need, workspace_bytes);
        return CSPN_ERR_WORKSPACE;
    }
    const long long hw = (long long)H * W;
    const uintptr_t n_f = span_bytes(B, C, hw), n_g = span_bytes(B, 9 * L, hw), n_o = span_bytes(B, C, L * hw);
    rc = check_disjoint({{feat, n_f, "feat"}, {gate, n_g, "gate"}, {out, n_o, "out"}, {grad_out, n_o, "grad_out"}},
                        {{grad_feat, n_f, "grad_feat"}, {grad_gate, n_g, "grad_gate"}, {workspace, need, "the workspace"}});
    if (rc != CSPN_OK) return rc;
    return on_device_of(feat, "feat", [&](int* launches) {
        return affinity_atrous_backward(feat, gate, out, grad_out, grad_feat, grad_gate, B, C, H, W, L, dilations, workspace,
                                        (cudaStream_t)stream, launches);
    });
}

// ---- 2D aggregation of the steps, K in {3, 5, 7} (DESIGN.md section 4.20): the K x K kernels of cspn2d_wide.cu at every K --
// The sizes, K, the norm, keep and the step list: true when they are valid (the error is set otherwise)
static bool agg_args_ok(int B, int C, int H, int W, int K, int gch, const int* steps, int n_steps, int norm_type, int keep) {
    if (!positive(B, C, H, W)) { set_error("non-positive shape B=%d C=%d H=%d W=%d", B, C, H, W); return false; }
    if (!kernel_size_ok(2, K)) { set_error("2D kernel size must be 3, 5 or 7, got %d", K); return false; }
    if (gch < K * K - 1) { set_error("a %dx%d kernel needs >= %d guidance channels, got %d", K, K, K * K - 1, gch); return false; }
    if (norm_type < 0 || norm_type > (int)CSPN_NORM_8SUM_ABS) { set_error("unknown norm_type %d", norm_type); return false; }
    if (keep != 0 && keep != 1) { set_error("keep must be 0 or 1, got %d", keep); return false; }
    if (n_steps < 1 || !steps) { set_error("the aggregation needs n_steps >= 1 and a step array, got %d", n_steps); return false; }
    for (int j = 0; j < n_steps; ++j)
        if (steps[j] < 1 || (j > 0 && steps[j] <= steps[j - 1])) {
            set_error("steps must be strictly increasing ints >= 1 (steps[%d]=%d)", j, steps[j]);
            return false;
        }
    return true;
}

// The alignment of the non-null pointers, the launch grid, the overlaps (`in` are read and `outs` written; null entries are
// absent buffers), then the workspace: the checks of an aggregation entry after its mandatory pointers and arguments
static int check_agg_buffers(int B, int C, std::vector<Buf> in, std::vector<Buf> outs, const void* ws, size_t ws_bytes,
                             size_t need) {
    uintptr_t bits = 0;
    for (auto* set : {&in, &outs}) {
        std::vector<Buf> kept;
        for (const Buf& b : *set)
            if (b.p) {
                bits |= reinterpret_cast<uintptr_t>(b.p);
                kept.push_back(b);
            }
        *set = kept;
    }
    if (bits & 3) { set_error("tensor pointers must be 4-byte aligned"); return CSPN_ERR_INVALID_ARGUMENT; }
    if ((long long)B * C > 65535) { set_error("2D aggregation: B*C=%lld exceeds gridDim.z", (long long)B * C); return CSPN_ERR_UNSUPPORTED; }
    const int rc = check_disjoint(in, outs);
    if (rc != CSPN_OK) return rc;
    if (!ws || ws_bytes < need) {
        set_error("2D aggregation needs %zu workspace bytes, got %zu", need, ws ? ws_bytes : (size_t)0);
        return CSPN_ERR_WORKSPACE;
    }
    return CSPN_OK;
}

size_t cspn2d_agg_workspace_bytes(int B, int C, int H, int W, int K, const int* steps, int n_steps, int keep) {
    if (!agg_args_ok(B, C, H, W, K, K * K - 1, steps, n_steps, 0, keep)) return 0;
    return aggregate2d_workspace_bytes(B, C, H, W, K, keep);
}

size_t cspn2d_agg_bwd_workspace_bytes(int B, int C, int H, int W, int K, const int* steps, int n_steps, int keep) {
    if (!agg_args_ok(B, C, H, W, K, K * K - 1, steps, n_steps, 0, keep)) return 0;
    return aggregate2d_bwd_workspace_bytes(B, C, H, W, K, steps[n_steps - 1], keep);
}

int cspn2d_agg_fwd_f32(const float* guidance, const float* blur, const float* sparse, const float* step_weight, float* out, int B,
                       int C, int H, int W, int guidance_channels, int K, const int* steps, int n_steps, int norm_type, int keep,
                       void* workspace, size_t workspace_bytes, cspn_stream_t stream) {
    begin_call();
    if (!guidance || !blur || !step_weight || !out) { set_error("null tensor pointer"); return CSPN_ERR_INVALID_ARGUMENT; }
    if (!agg_args_ok(B, C, H, W, K, guidance_channels, steps, n_steps, norm_type, keep)) return CSPN_ERR_INVALID_ARGUMENT;
    const long long hw = (long long)H * W;
    const size_t need = aggregate2d_workspace_bytes(B, C, H, W, K, keep && sparse);
    const int rc = check_agg_buffers(B, C,
                                     {{guidance, span_bytes(B, guidance_channels, hw), "guidance"}, {blur, span_bytes(B, C, hw), "blur"},
                                      {sparse, span_bytes(B, 1, hw), "sparse"}, {step_weight, span_bytes(B, n_steps, hw), "step_weight"}},
                                     {{out, span_bytes(B, C, hw), "out"}, {workspace, need, "the workspace"}}, workspace,
                                     workspace_bytes, need);
    if (rc != CSPN_OK) return rc;
    return on_device_of(blur, "blur", [&](int* launches) {
        Problem2D p{guidance, blur, sparse, out, B, C, H, W, guidance_channels, steps[n_steps - 1], norm_type == CSPN_NORM_8SUM_ABS};
        p.keep = keep && sparse;
        return aggregate2d_forward(p, K, step_weight, steps, n_steps, workspace, workspace_bytes, (cudaStream_t)stream, launches);
    });
}

int cspn2d_agg_bwd_f32(const float* guidance, const float* blur, const float* sparse, const float* step_weight, const float* grad_out,
                       float* grad_guidance, float* grad_blur, float* grad_sparse, float* grad_step_weight, int B, int C, int H,
                       int W, int guidance_channels, int K, const int* steps, int n_steps, int norm_type, int keep, void* workspace,
                       size_t workspace_bytes, cspn_stream_t stream) {
    begin_call();
    if (!guidance || !blur || !step_weight || !grad_out) { set_error("null tensor pointer"); return CSPN_ERR_INVALID_ARGUMENT; }
    if (!agg_args_ok(B, C, H, W, K, guidance_channels, steps, n_steps, norm_type, keep)) return CSPN_ERR_INVALID_ARGUMENT;
    const long long hw = (long long)H * W;
    const uintptr_t n_g = span_bytes(B, guidance_channels, hw), n_d = span_bytes(B, C, hw), n_s = span_bytes(B, 1, hw),
                    n_w = span_bytes(B, n_steps, hw);
    const size_t need = aggregate2d_bwd_workspace_bytes(B, C, H, W, K, steps[n_steps - 1], keep && sparse);
    const int rc = check_agg_buffers(B, C,
                                     {{guidance, n_g, "guidance"}, {blur, n_d, "blur"}, {sparse, n_s, "sparse"},
                                      {step_weight, n_w, "step_weight"}, {grad_out, n_d, "grad_out"}},
                                     {{grad_guidance, n_g, "grad_guidance"}, {grad_blur, n_d, "grad_blur"},
                                      {grad_sparse, n_s, "grad_sparse"}, {grad_step_weight, n_w, "grad_step_weight"},
                                      {workspace, need, "the workspace"}},
                                     workspace, workspace_bytes, need);
    if (rc != CSPN_OK) return rc;
    return on_device_of(blur, "blur", [&](int* launches) -> int {
        Problem2D p{guidance, blur, sparse, nullptr, B, C, H, W, guidance_channels, steps[n_steps - 1], norm_type == CSPN_NORM_8SUM_ABS};
        p.keep = keep && sparse;
        // the default mode's m = sign(sparse) is not differentiated (Affinity_PropagateK detaches it); no samples, no gradient
        if (grad_sparse && !p.keep)
            CSPN_CUDA_TRY(cudaMemsetAsync(grad_sparse, 0, (size_t)B * H * W * sizeof(float), (cudaStream_t)stream));
        return aggregate2d_backward(p, K, step_weight, steps, n_steps, grad_out, grad_guidance, grad_blur, p.keep ? grad_sparse : nullptr,
                                    grad_step_weight, workspace, workspace_bytes, (cudaStream_t)stream, launches);
    });
}

// ---- 2D non-local propagation, NLSPN's (DESIGN.md section 4.21): cspn2d_nonlocal.cu ----------------------------------------
// The sizes, K and the step count: true when they are valid (the error is set otherwise)
static bool nl_args_ok(int B, int C, int H, int W, int K, int iters) {
    if (!positive(B, C, H, W)) { set_error("non-positive shape B=%d C=%d H=%d W=%d", B, C, H, W); return false; }
    if (!kernel_size_ok(2, K)) { set_error("2D kernel size must be 3, 5 or 7, got %d", K); return false; }
    if (iters < 0) { set_error("prop_time must be >= 0, got %d", iters); return false; }
    return true;
}

// The alignment of the non-null pointers, the launch limits, the overlaps (`in` are read and `outs` written; null entries
// are absent buffers), then the workspace (none needed when need is 0)
static int check_nl_buffers(int B, int C, int H, int W, int K, std::vector<Buf> in, std::vector<Buf> outs, const void* ws,
                            size_t ws_bytes, size_t need) {
    uintptr_t bits = 0;
    for (auto* set : {&in, &outs}) {
        std::vector<Buf> kept;
        for (const Buf& b : *set)
            if (b.p) {
                bits |= reinterpret_cast<uintptr_t>(b.p);
                kept.push_back(b);
            }
        *set = kept;
    }
    if (bits & 3) { set_error("tensor pointers must be 4-byte aligned"); return CSPN_ERR_INVALID_ARGUMENT; }
    const char* why = "";
    if (!nonlocal2d_launchable(B, C, H, W, K, &why)) { set_error("unsupported shape: %s", why); return CSPN_ERR_UNSUPPORTED; }
    const int rc = check_disjoint(in, outs);
    if (rc != CSPN_OK) return rc;
    if (need && (!ws || ws_bytes < need)) {
        set_error("the non-local propagation needs %zu workspace bytes, got %zu", need, ws ? ws_bytes : (size_t)0);
        return CSPN_ERR_WORKSPACE;
    }
    return CSPN_OK;
}

size_t cspn2d_nl_workspace_bytes(int B, int C, int H, int W, int K, int iters) {
    if (!nl_args_ok(B, C, H, W, K, iters)) return 0;
    return nonlocal2d_workspace_bytes(B, C, H, W, iters);
}

size_t cspn2d_nl_bwd_workspace_bytes(int B, int C, int H, int W, int K, int iters) {
    if (!nl_args_ok(B, C, H, W, K, iters)) return 0;
    const char* why = "";
    if (!nonlocal2d_launchable(B, C, H, W, K, &why)) return 0;
    return nonlocal2d_bwd_workspace_bytes(B, C, H, W, K, iters);
}

int cspn2d_nl_fwd_f32(const float* feat, const float* offset, const float* affinity, const float* sparse, float* out, int B, int C,
                      int H, int W, int K, int iters, void* workspace, size_t workspace_bytes, cspn_stream_t stream) {
    begin_call();
    if (!feat || !offset || !affinity || !out) { set_error("null tensor pointer"); return CSPN_ERR_INVALID_ARGUMENT; }
    if (!nl_args_ok(B, C, H, W, K, iters)) return CSPN_ERR_INVALID_ARGUMENT;
    const long long hw = (long long)H * W, T = (long long)K * K - 1;
    const uintptr_t n_f = span_bytes(B, C, hw);
    const size_t need = nonlocal2d_workspace_bytes(B, C, H, W, iters);
    const int rc = check_nl_buffers(B, C, H, W, K,
                                    {{feat, n_f, "feat"}, {offset, span_bytes(B, (int)(2 * T), hw), "offset"},
                                     {affinity, span_bytes(B, (int)T, hw), "affinity"}, {sparse, n_f, "sparse"}},
                                    {{out, n_f, "out"}, {need ? workspace : nullptr, need, "the workspace"}}, workspace,
                                    workspace_bytes, need);
    if (rc != CSPN_OK) return rc;
    return on_device_of(feat, "feat", [&](int* launches) {
        return nonlocal2d_forward(feat, offset, affinity, sparse, out, B, C, H, W, K, iters, workspace, (cudaStream_t)stream, launches);
    });
}

int cspn2d_nl_bwd_f32(const float* feat, const float* offset, const float* affinity, const float* sparse, const float* grad_out,
                      float* grad_feat, float* grad_offset, float* grad_affinity, float* grad_sparse, int B, int C, int H, int W, int K,
                      int iters, void* workspace, size_t workspace_bytes, cspn_stream_t stream) {
    begin_call();
    if (!feat || !offset || !affinity || !grad_out) { set_error("null tensor pointer"); return CSPN_ERR_INVALID_ARGUMENT; }
    if (!nl_args_ok(B, C, H, W, K, iters)) return CSPN_ERR_INVALID_ARGUMENT;
    if (grad_sparse && !sparse) { set_error("grad_sparse needs a sparse input"); return CSPN_ERR_INVALID_ARGUMENT; }
    const long long hw = (long long)H * W, T = (long long)K * K - 1;
    const uintptr_t n_f = span_bytes(B, C, hw), n_o = span_bytes(B, (int)(2 * T), hw), n_a = span_bytes(B, (int)T, hw);
    const std::vector<Buf> in{{feat, n_f, "feat"}, {offset, n_o, "offset"}, {affinity, n_a, "affinity"}, {sparse, n_f, "sparse"},
                              {grad_out, n_f, "grad_out"}};
    const std::vector<Buf> outs{{grad_feat, n_f, "grad_feat"}, {grad_offset, n_o, "grad_offset"}, {grad_affinity, n_a, "grad_affinity"},
                                {grad_sparse, n_f, "grad_sparse"}};
    int rc = check_nl_buffers(B, C, H, W, K, in, outs, nullptr, 0, 0);
    if (rc != CSPN_OK) return rc;
    // the radix sort sizes its scratch for the current device's architecture: the one query that needs the CUDA runtime
    const size_t need = iters > 0 ? nonlocal2d_bwd_workspace_bytes(B, C, H, W, K, iters) : 0;
    if (iters > 0 && need == 0) { set_error("cannot size the backward's workspace (no CUDA device?)"); return CSPN_ERR_CUDA; }
    if (need) {
        std::vector<Buf> all;
        for (const Buf& b : in) if (b.p) all.push_back(b);
        for (const Buf& b : outs) if (b.p) all.push_back(b);
        rc = check_nl_buffers(B, C, H, W, K, all, {{workspace, need, "the workspace"}}, workspace, workspace_bytes, need);
        if (rc != CSPN_OK) return rc;
    }
    return on_device_of(feat, "feat", [&](int* launches) {
        return nonlocal2d_backward(feat, offset, affinity, sparse, grad_out, grad_feat, grad_offset, grad_affinity, grad_sparse, B, C,
                                   H, W, K, iters, workspace, (cudaStream_t)stream, launches);
    });
}

// ---- 2D dilated propagation with a centre weight and a learned confidence, PENet's DA-CSPN++ (DESIGN.md section 4.22) ------
// The sizes, K, the dilation and the step count: true when they are valid (the error is set otherwise)
static bool dil_args_ok(int B, int C, int H, int W, int K, int dilation, int iters) {
    if (!positive(B, C, H, W)) { set_error("non-positive shape B=%d C=%d H=%d W=%d", B, C, H, W); return false; }
    if (!kernel_size_ok(2, K)) { set_error("2D kernel size must be 3, 5 or 7, got %d", K); return false; }
    if (dilation < 1 || dilation > 4) { set_error("dilation must be in [1, 4], got %d", dilation); return false; }
    if (iters < 0) { set_error("prop_time must be >= 0, got %d", iters); return false; }
    return true;
}

// The alignment of the non-null pointers, the launch limits, the overlaps (`in` are read and `outs` written; null entries
// are absent buffers), then the workspace.  Shared by the dilated and the dynamic propagation (`what`, `launchable`).
static int check_dil_buffers(int B, int C, int H, int W, std::vector<Buf> in, std::vector<Buf> outs, const void* ws, size_t ws_bytes,
                             size_t need, const char* what = "the dilated propagation",
                             int (*launchable)(int, int, int, int, const char**) = dilated2d_launchable) {
    uintptr_t bits = 0;
    for (auto* set : {&in, &outs}) {
        std::vector<Buf> kept;
        for (const Buf& b : *set)
            if (b.p) {
                bits |= reinterpret_cast<uintptr_t>(b.p);
                kept.push_back(b);
            }
        *set = kept;
    }
    if (bits & 3) { set_error("tensor pointers must be 4-byte aligned"); return CSPN_ERR_INVALID_ARGUMENT; }
    const char* why = "";
    if (!launchable(B, C, H, W, &why)) { set_error("unsupported shape: %s", why); return CSPN_ERR_UNSUPPORTED; }
    const int rc = check_disjoint(in, outs);
    if (rc != CSPN_OK) return rc;
    if (need && (!ws || ws_bytes < need)) {
        set_error("%s needs %zu workspace bytes, got %zu", what, need, ws ? ws_bytes : (size_t)0);
        return CSPN_ERR_WORKSPACE;
    }
    return CSPN_OK;
}

size_t cspn2d_dil_workspace_bytes(int B, int C, int H, int W, int K, int dilation, int iters) {
    if (!dil_args_ok(B, C, H, W, K, dilation, iters)) return 0;
    return dilated2d_workspace_bytes(B, C, H, W, iters);
}

size_t cspn2d_dil_bwd_workspace_bytes(int B, int C, int H, int W, int K, int dilation, int iters) {
    if (!dil_args_ok(B, C, H, W, K, dilation, iters)) return 0;
    return dilated2d_bwd_workspace_bytes(B, C, H, W, iters);
}

int cspn2d_dil_fwd_f32(const float* kernel, const float* blur, const float* sparse, const float* confidence, float* out, int B, int C,
                       int H, int W, int K, int dilation, int iters, void* workspace, size_t workspace_bytes, cspn_stream_t stream) {
    begin_call();
    if (!kernel || !blur || !out) { set_error("null tensor pointer"); return CSPN_ERR_INVALID_ARGUMENT; }
    if (!sparse != !confidence) { set_error("sparse and confidence come together or not at all"); return CSPN_ERR_INVALID_ARGUMENT; }
    if (!dil_args_ok(B, C, H, W, K, dilation, iters)) return CSPN_ERR_INVALID_ARGUMENT;
    const long long hw = (long long)H * W;
    const uintptr_t n_b = span_bytes(B, C, hw), n_1 = span_bytes(B, 1, hw);
    const size_t need = dilated2d_workspace_bytes(B, C, H, W, iters);
    const int rc = check_dil_buffers(B, C, H, W,
                                     {{kernel, span_bytes(B, K * K, hw), "kernel"}, {blur, n_b, "blur"}, {sparse, n_1, "sparse"},
                                      {confidence, n_1, "confidence"}},
                                     {{out, n_b, "out"}, {need ? workspace : nullptr, need, "the workspace"}}, workspace, workspace_bytes,
                                     need);
    if (rc != CSPN_OK) return rc;
    return on_device_of(blur, "blur", [&](int* launches) {
        return dilated2d_forward(kernel, blur, sparse, confidence, out, B, C, H, W, K, dilation, iters, workspace, (cudaStream_t)stream,
                                 launches);
    });
}

int cspn2d_dil_bwd_f32(const float* kernel, const float* blur, const float* sparse, const float* confidence, const float* grad_out,
                       float* grad_kernel, float* grad_blur, float* grad_sparse, float* grad_confidence, int B, int C, int H, int W,
                       int K, int dilation, int iters, void* workspace, size_t workspace_bytes, cspn_stream_t stream) {
    begin_call();
    if (!kernel || !blur || !grad_out) { set_error("null tensor pointer"); return CSPN_ERR_INVALID_ARGUMENT; }
    if (!sparse != !confidence) { set_error("sparse and confidence come together or not at all"); return CSPN_ERR_INVALID_ARGUMENT; }
    if ((grad_sparse || grad_confidence) && !sparse) {
        set_error("grad_sparse and grad_confidence need the samples");
        return CSPN_ERR_INVALID_ARGUMENT;
    }
    if (!dil_args_ok(B, C, H, W, K, dilation, iters)) return CSPN_ERR_INVALID_ARGUMENT;
    const long long hw = (long long)H * W;
    const uintptr_t n_b = span_bytes(B, C, hw), n_1 = span_bytes(B, 1, hw), n_k = span_bytes(B, K * K, hw);
    const size_t need = dilated2d_bwd_workspace_bytes(B, C, H, W, iters);
    const int rc = check_dil_buffers(
            B, C, H, W,
            {{kernel, n_k, "kernel"}, {blur, n_b, "blur"}, {sparse, n_1, "sparse"}, {confidence, n_1, "confidence"},
             {grad_out, n_b, "grad_out"}},
            {{grad_kernel, n_k, "grad_kernel"}, {grad_blur, n_b, "grad_blur"}, {grad_sparse, n_1, "grad_sparse"},
             {grad_confidence, n_1, "grad_confidence"}, {need ? workspace : nullptr, need, "the workspace"}},
            workspace, workspace_bytes, need);
    if (rc != CSPN_OK) return rc;
    return on_device_of(blur, "blur", [&](int* launches) {
        return dilated2d_backward(kernel, blur, sparse, confidence, grad_out, grad_kernel, grad_blur, grad_sparse, grad_confidence, B, C,
                                  H, W, K, dilation, iters, workspace, (cudaStream_t)stream, launches);
    });
}

// ---- 2D dynamic propagation with per-step ring attention and an anchor to d_0, DySPN's step (DESIGN.md section 4.23) -------
static bool dyn_args_ok(int B, int C, int H, int W, int K, int iters) {
    if (!positive(B, C, H, W)) { set_error("non-positive shape B=%d C=%d H=%d W=%d", B, C, H, W); return false; }
    if (!kernel_size_ok(2, K)) { set_error("2D kernel size must be 3, 5 or 7, got %d", K); return false; }
    if (iters < 0) { set_error("the step count must be >= 0, got %d", iters); return false; }
    if ((long long)iters * ((K + 1) / 2) > INT32_MAX) { set_error("iters * (K + 1) / 2 attention channels exceed 2^31 - 1"); return false; }
    return true;
}

size_t cspn2d_dyn_workspace_bytes(int B, int C, int H, int W, int K, int iters) {
    if (!dyn_args_ok(B, C, H, W, K, iters)) return 0;
    return dynamic2d_workspace_bytes(B, C, H, W, iters);
}

size_t cspn2d_dyn_bwd_workspace_bytes(int B, int C, int H, int W, int K, int iters) {
    if (!dyn_args_ok(B, C, H, W, K, iters)) return 0;
    return dynamic2d_bwd_workspace_bytes(B, C, H, W, iters);
}

int cspn2d_dyn_fwd_f32(const float* affinity, const float* attention, const float* blur, const float* sparse, const float* confidence,
                       float* out, int B, int C, int H, int W, int K, int iters, void* workspace, size_t workspace_bytes,
                       cspn_stream_t stream) {
    begin_call();
    if (!affinity || !blur || !out || (!attention && iters > 0)) { set_error("null tensor pointer"); return CSPN_ERR_INVALID_ARGUMENT; }
    if (!sparse != !confidence) { set_error("sparse and confidence come together or not at all"); return CSPN_ERR_INVALID_ARGUMENT; }
    if (!dyn_args_ok(B, C, H, W, K, iters)) return CSPN_ERR_INVALID_ARGUMENT;
    const long long hw = (long long)H * W;
    const uintptr_t n_b = span_bytes(B, C, hw), n_1 = span_bytes(B, 1, hw);
    const size_t need = dynamic2d_workspace_bytes(B, C, H, W, iters);
    const int rc = check_dil_buffers(B, C, H, W,
                                     {{affinity, span_bytes(B, K * K, hw), "affinity"},
                                      {iters ? attention : nullptr, span_bytes(B, iters * ((K + 1) / 2), hw), "attention"},
                                      {blur, n_b, "blur"}, {sparse, n_1, "sparse"}, {confidence, n_1, "confidence"}},
                                     {{out, n_b, "out"}, {need ? workspace : nullptr, need, "the workspace"}}, workspace, workspace_bytes,
                                     need, "the dynamic propagation", dynamic2d_launchable);
    if (rc != CSPN_OK) return rc;
    return on_device_of(blur, "blur", [&](int* launches) {
        return dynamic2d_forward(affinity, attention, blur, sparse, confidence, out, B, C, H, W, K, iters, workspace, (cudaStream_t)stream,
                                 launches);
    });
}

int cspn2d_dyn_bwd_f32(const float* affinity, const float* attention, const float* blur, const float* sparse, const float* confidence,
                       const float* grad_out, float* grad_affinity, float* grad_attention, float* grad_blur, float* grad_sparse,
                       float* grad_confidence, int B, int C, int H, int W, int K, int iters, void* workspace, size_t workspace_bytes,
                       cspn_stream_t stream) {
    begin_call();
    if (!affinity || !blur || !grad_out || (!attention && iters > 0)) {
        set_error("null tensor pointer");
        return CSPN_ERR_INVALID_ARGUMENT;
    }
    if (!sparse != !confidence) { set_error("sparse and confidence come together or not at all"); return CSPN_ERR_INVALID_ARGUMENT; }
    if ((grad_sparse || grad_confidence) && !sparse) {
        set_error("grad_sparse and grad_confidence need the samples");
        return CSPN_ERR_INVALID_ARGUMENT;
    }
    if (!dyn_args_ok(B, C, H, W, K, iters)) return CSPN_ERR_INVALID_ARGUMENT;
    const long long hw = (long long)H * W;
    const uintptr_t n_b = span_bytes(B, C, hw), n_1 = span_bytes(B, 1, hw), n_k = span_bytes(B, K * K, hw);
    const uintptr_t n_a = span_bytes(B, iters * ((K + 1) / 2), hw);
    const size_t need = dynamic2d_bwd_workspace_bytes(B, C, H, W, iters);
    const int rc = check_dil_buffers(
            B, C, H, W,
            {{affinity, n_k, "affinity"}, {iters ? attention : nullptr, n_a, "attention"}, {blur, n_b, "blur"}, {sparse, n_1, "sparse"},
             {confidence, n_1, "confidence"}, {grad_out, n_b, "grad_out"}},
            {{grad_affinity, n_k, "grad_affinity"}, {iters ? grad_attention : nullptr, n_a, "grad_attention"}, {grad_blur, n_b, "grad_blur"},
             {grad_sparse, n_1, "grad_sparse"}, {grad_confidence, n_1, "grad_confidence"}, {need ? workspace : nullptr, need, "the workspace"}},
            workspace, workspace_bytes, need, "the dynamic propagation", dynamic2d_launchable);
    if (rc != CSPN_OK) return rc;
    return on_device_of(blur, "blur", [&](int* launches) {
        return dynamic2d_backward(affinity, attention, blur, sparse, confidence, grad_out, grad_affinity, iters ? grad_attention : nullptr,
                                  grad_blur, grad_sparse, grad_confidence, B, C, H, W, K, iters, workspace, (cudaStream_t)stream, launches);
    });
}

// ---- 2D linear three-way scans, SPN's propagation (DESIGN.md section 4.24) -------------------------------------------
static bool lin_args_ok(int B, int C, int H, int W, int mask, int gate_mode) {
    if (!positive(B, C, H, W)) { set_error("non-positive shape B=%d C=%d H=%d W=%d", B, C, H, W); return false; }
    if (mask < 1 || mask > 15) { set_error("dir_mask must be 1 .. 15 (bits l2r, r2l, t2b, b2t), got %d", mask); return false; }
    if (gate_mode != CSPN_LIN_GATE_SHARED && gate_mode != CSPN_LIN_GATE_PER_CHANNEL) {
        set_error("unknown gate_mode %d", gate_mode);
        return false;
    }
    if ((long long)3 * __builtin_popcount(mask) * (gate_mode ? C : 1) > INT32_MAX) { set_error("3 * nd * C gate channels exceed 2^31 - 1"); return false; }
    return true;
}

// The alignment of the non-null pointers, the launch limits, the overlaps, then the workspace
static int check_lin_buffers(int B, int C, int H, int W, int mask, std::vector<Buf> in, std::vector<Buf> outs, const void* ws,
                             size_t ws_bytes, size_t need) {
    uintptr_t bits = 0;
    for (auto* set : {&in, &outs}) {
        std::vector<Buf> kept;
        for (const Buf& b : *set)
            if (b.p) {
                bits |= reinterpret_cast<uintptr_t>(b.p);
                kept.push_back(b);
            }
        *set = kept;
    }
    if (bits & 3) { set_error("tensor pointers must be 4-byte aligned"); return CSPN_ERR_INVALID_ARGUMENT; }
    const char* why = "";
    if (!linear2d_launchable(B, C, H, W, mask, &why)) { set_error("unsupported shape: %s", why); return CSPN_ERR_UNSUPPORTED; }
    const int rc = check_disjoint(in, outs);
    if (rc != CSPN_OK) return rc;
    if (need && (!ws || ws_bytes < need)) {
        set_error("the linear propagation needs %zu workspace bytes, got %zu", need, ws ? ws_bytes : (size_t)0);
        return CSPN_ERR_WORKSPACE;
    }
    return CSPN_OK;
}

size_t cspn2d_lin_workspace_bytes(int B, int C, int H, int W, int dir_mask, int gate_mode) {
    if (!lin_args_ok(B, C, H, W, dir_mask, gate_mode)) return 0;
    return linear2d_workspace_bytes(B, C, H, W, dir_mask);
}

size_t cspn2d_lin_bwd_workspace_bytes(int B, int C, int H, int W, int dir_mask, int gate_mode) {
    if (!lin_args_ok(B, C, H, W, dir_mask, gate_mode)) return 0;
    return linear2d_bwd_workspace_bytes(B, C, H, W, dir_mask, gate_mode ? C : 1);
}

int cspn2d_lin_fwd_f32(const float* feat, const float* gate, float* out, float* planes, int B, int C, int H, int W, int dir_mask,
                       int gate_mode, void* workspace, size_t workspace_bytes, cspn_stream_t stream) {
    begin_call();
    if (!feat || !gate || !out) { set_error("null tensor pointer"); return CSPN_ERR_INVALID_ARGUMENT; }
    if (!lin_args_ok(B, C, H, W, dir_mask, gate_mode)) return CSPN_ERR_INVALID_ARGUMENT;
    const int nd = __builtin_popcount(dir_mask), Cg = gate_mode ? C : 1;
    if (planes && nd == 1) { set_error("planes must be NULL for one direction (its plane is out)"); return CSPN_ERR_INVALID_ARGUMENT; }
    const long long hw = (long long)H * W;
    const uintptr_t n_x = span_bytes(B, C, hw), n_p = span_bytes(B, C, nd * hw);
    const size_t need = planes ? 0 : linear2d_workspace_bytes(B, C, H, W, dir_mask);
    float* pl = nd > 1 ? (planes ? planes : static_cast<float*>(workspace)) : nullptr;
    const int rc = check_lin_buffers(B, C, H, W, dir_mask, {{feat, n_x, "feat"}, {gate, span_bytes(B, 3 * nd * Cg, hw), "gate"}},
                                     {{out, n_x, "out"}, {planes, n_p, "planes"}, {need ? workspace : nullptr, need, "the workspace"}},
                                     workspace, workspace_bytes, need);
    if (rc != CSPN_OK) return rc;
    return on_device_of(feat, "feat", [&](int* launches) {
        return linear2d_forward(feat, gate, out, pl, B, C, H, W, dir_mask, Cg, (cudaStream_t)stream, launches);
    });
}

int cspn2d_lin_bwd_f32(const float* feat, const float* gate, const float* planes, const float* grad_out, float* grad_feat,
                       float* grad_gate, int B, int C, int H, int W, int dir_mask, int gate_mode, void* workspace, size_t workspace_bytes,
                       cspn_stream_t stream) {
    begin_call();
    if (!feat || !gate || !planes || !grad_out) { set_error("null tensor pointer"); return CSPN_ERR_INVALID_ARGUMENT; }
    if (!lin_args_ok(B, C, H, W, dir_mask, gate_mode)) return CSPN_ERR_INVALID_ARGUMENT;
    const int nd = __builtin_popcount(dir_mask), Cg = gate_mode ? C : 1;
    const long long hw = (long long)H * W;
    const uintptr_t n_x = span_bytes(B, C, hw), n_g = span_bytes(B, 3 * nd * Cg, hw);
    const size_t need = (grad_feat || grad_gate) ? linear2d_bwd_workspace_bytes(B, C, H, W, dir_mask, Cg) : 0;
    const int rc = check_lin_buffers(B, C, H, W, dir_mask,
                                     {{feat, n_x, "feat"}, {gate, n_g, "gate"}, {planes, span_bytes(B, C, nd * hw), "planes"},
                                      {grad_out, n_x, "grad_out"}},
                                     {{grad_feat, n_x, "grad_feat"}, {grad_gate, n_g, "grad_gate"}, {need ? workspace : nullptr, need, "the workspace"}},
                                     workspace, workspace_bytes, need);
    if (rc != CSPN_OK) return rc;
    return on_device_of(feat, "feat", [&](int* launches) {
        return linear2d_backward(feat, gate, planes, grad_out, grad_feat, grad_gate, B, C, H, W, dir_mask, Cg, workspace,
                                 (cudaStream_t)stream, launches);
    });
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

static int plan_json(int H, int W, int iters, int chained, char* buf, int buf_len) {
    if (!buf || buf_len <= 0) return 0;
    if (!positive(H, W, iters)) return snprintf(buf, buf_len, "{\"supported\": false, \"why\": \"invalid shape\"}");
    return cluster2d_plan_json(H, W, iters, chained, buf, buf_len);
}

int cspn2d_plan_json(int H, int W, int iters, char* buf, int buf_len) { return plan_json(H, W, iters, 0, buf, buf_len); }

int cspn2d_plan_json_chained(int H, int W, int iters, char* buf, int buf_len) { return plan_json(H, W, iters, 1, buf, buf_len); }

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
    begin_call();
    int rc = check_prop(2, guidance, blur, out, B, C, 1, H, W, 3, guidance_channels, iters, norm_type);
    if (rc == CSPN_OK) rc = check_algo(algo);
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
    begin_call();
    if (const int rc = check_prop(3, guidance, feat, out, B, C, D, H, W, 3, 0, iters, norm_type)) return rc;
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
