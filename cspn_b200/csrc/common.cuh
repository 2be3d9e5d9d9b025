// Shared declarations of the cspn_b200 native library (sm_90a only).
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>

#include <cstdarg>
#include <cstddef>
#include <cstdint>
#include <cstdio>

#include "../../include/cspn_b200.h"

namespace cspn {

// ---- thread-local status -------------------------------------------------------------------
void set_error(const char* fmt, ...);
void clear_error();
extern thread_local int g_last_algo;
extern thread_local int g_last_launches;

#define CSPN_CUDA_TRY(expr)                                                                     \
    do {                                                                                        \
        cudaError_t _e = (expr);                                                                \
        if (_e != cudaSuccess) {                                                                \
            ::cspn::set_error("%s failed: %s (%s:%d)", #expr, cudaGetErrorString(_e), __FILE__, \
                              __LINE__);                                                        \
            return CSPN_ERR_CUDA;                                                               \
        }                                                                                       \
    } while (0)

// (dy,dx) that guidance channel k / depth copy k is read from.  Derived from the ZeroPad2d
// tuples at /root/reference/cspn_pytorch/models/cspn.py:105-129 (= :149-168) and the crop at
// :72,:142: pad (l,r,t,b) then [1:-1,1:-1] reads the source at (y+1-t, x+1-l).
//   k : 0       1      2       3      4       5       6       7
//      (+1,+1) (+1,0) (+1,-1) (0,+1) (0,-1) (-1,+1) (-1,0) (-1,-1)
__host__ __device__ constexpr int off2_dy(int k) { return k < 3 ? 1 : (k < 5 ? 0 : -1); }
__host__ __device__ constexpr int off2_dx(int k) {
    return k < 3 ? 1 - k : (k == 3 ? 1 : (k == 4 ? -1 : 6 - k));
}
// 3D: raster order over pad triples (f,t,l) in {0,1,2}^3 minus the centre; offset = 1 - pad.
__host__ __device__ constexpr int off3_idx(int k) { return k >= 13 ? k + 1 : k; }
__host__ __device__ constexpr int off3_dz(int k) { return 1 - off3_idx(k) / 9; }
__host__ __device__ constexpr int off3_dy(int k) { return 1 - (off3_idx(k) / 3) % 3; }
__host__ __device__ constexpr int off3_dx(int k) { return 1 - off3_idx(k) % 3; }

__device__ __forceinline__ float signf(float v) { return (v > 0.f ? 1.f : 0.f) - (v < 0.f ? 1.f : 0.f); }

// a sum of |gates| whose quotient form must be used: 0 (0/0 = NaN), subnormal (divided exactly), inf or NaN (weights 0 / NaN)
__device__ __forceinline__ bool cold_sum(float S) { return !(S >= 1.17549435e-38f && S <= 3.40282347e38f); }
// The own-location ('paddle') steps divide acc = sum_k |g_k| d(p + off_k) by S once.  That is the quotient form
// sum_k (|g_k| / S) d(p + off_k) up to rounding only where S is normal and acc finite: an acc that overflowed (a large S
// times |d| > 1) or met an inf / NaN of d must be formed from the quotients too, so that each term is w_k d as the weights have it
__device__ __forceinline__ bool cold_paddle(float S, float acc) { return cold_sum(S) || !(fabsf(acc) <= 3.40282347e38f); }

// ---- problem descriptors --------------------------------------------------------------------
struct Problem2D {
    const float* guidance;  // [B][gch][H][W]
    const float* blur;      // [B][C][H][W]
    const float* sparse;    // [B][1][H][W] or nullptr
    float* out;             // [B][C][H][W]
    int B, C, H, W, gch, iters, norm_abs;
    int keep = 0;           // keep the sparse samples (DESIGN.md section 4.13): m = 1[sparse > 0], replaced by sparse itself
};

// ---- per-algorithm launchers (each returns a cspn_status; enqueue only, no sync) -------------
// keep: the keep-sparse mode, which needs one more B*C*H*W plane (d0', see launch_prep_keep)
size_t generic2d_workspace_bytes(int B, int C, int H, int W, int iters, bool keep = false);
int generic2d_forward(const Problem2D& p, void* ws, size_t ws_bytes, cudaStream_t stream, int* launches);

// ws: the caller's workspace (nullptr when not known yet); a plan of several passes keeps its intermediate result there
// with float4 stores and loads, so it declines a workspace that is not 16-byte aligned
bool cluster2d_supported(const Problem2D& p, char* why, int why_len, const void* ws = nullptr);
size_t cluster2d_workspace_bytes(int B, int C, int H, int W, int iters);
// peer_out / mc_out: additional destinations of the final result (fused gather), see cspn2d_fwd_gather_f32
int cluster2d_forward(const Problem2D& p, void* ws, size_t ws_bytes, cudaStream_t stream, int* launches,
                      float* const* peer_out = nullptr, int n_peer = 0, float* mc_out = nullptr);
int cluster2d_describe(int B, int C, int H, int W, int iters, char* buf, int len);
int cluster2d_plan_json(int H, int W, int iters, int chained, char* buf, int len);
// staged (opt-in, see cspn2d_bwd.cu): the forward keeping every iterate, and the adjoint sweep, on the cluster kernel
int cluster2d_forward_steps(const Problem2D& p, float* steps, cudaStream_t stream, int* launches);
int cluster2d_adjoint_steps(const Problem2D& p, const float* grad_out, float* lam, cudaStream_t stream, int* launches);

// Keep-sparse prep of the K x K and 3x3 launch-per-step paths (cspn2d_wide.cu): the K*K planes of prep2d_kernel /
// prepk_kernel with m = 1[sparse > 0] (w'_k, kappa), and d0 [B][C][H][W] = (1-m) blur + m sparse, the value the constant
// term kappa * d0 of the unchanged step kernels multiplies
void launch_prep_keep(int K, const float* guidance, const float* sparse, const float* blur, float* wk, float* d0, int B, int C,
                      int H, int W, int gch, int norm_abs, cudaStream_t stream);

// The 3x3 backward: the cluster formulation, else the K x K one at K = 3 (cspn2d_bwd.cu).  keep: as for
// generic2d_workspace_bytes.  grad_sparse: [B][1][H][W], written in keep mode only (may be null)
size_t bwd2d_workspace_bytes(int B, int C, int H, int W, int iters, bool keep = false);
int bwd2d(const Problem2D& p, const float* grad_out, float* grad_guidance, float* grad_blur, void* ws,
          size_t ws_bytes, cudaStream_t stream, int* launches, float* grad_sparse = nullptr);

// Fused gather of the K x K, 'paddle' and gates forwards (cspn2d_{k,paddle,gates}_fwd_gather_f32): the last step also
// stores its result to these destinations, each addressed like p.out -- up to 7 peer-mapped bases (NVLink stores) and one
// NVLS multicast base or null; all 16-byte aligned.  Passed by value to the step kernel (the Scatter of cspn2d_cluster.cu).
struct Fan {
    float* peer[7];
    int n_peer;
    float* mc;
};

// The destinations of fan moved `off` floats on, as `out` is for a launch group that starts `off` floats into it
inline Fan offset_fan(const Fan& f, size_t off) {
    Fan g{};
    g.n_peer = f.n_peer;
    for (int e = 0; e < f.n_peer; ++e) g.peer[e] = f.peer[e] + off;
    g.mc = f.mc ? f.mc + off : nullptr;
    return g;
}

// The FAN epilogue of the step kernels: v, just stored at element o of dst, also to element o of every destination
__device__ __forceinline__ void fan_store(const Fan& fan, size_t o, float4 v) {
#pragma unroll
    for (int e = 0; e < 7; ++e)          // peer GPUs' gather buffers (NVLink stores); n_peer is uniform
        if (e < fan.n_peer) __stcs(reinterpret_cast<float4*>(fan.peer[e] + o), v);
    if (fan.mc)                          // NVLS: one store, replicated by the switch
        asm volatile("multimem.st.relaxed.sys.global.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(fan.mc + o), "f"(v.x), "f"(v.y),
                     "f"(v.z), "f"(v.w) : "memory");
}

__device__ __forceinline__ void fan_store(const Fan& fan, size_t o, float v) {
#pragma unroll
    for (int e = 0; e < 7; ++e)
        if (e < fan.n_peer) __stcs(fan.peer[e] + o, v);
    if (fan.mc) asm volatile("multimem.st.relaxed.sys.global.f32 [%0], %1;" ::"l"(fan.mc + o), "f"(v) : "memory");
}

// The operator families of the wide kernels (cspn2d_wide.cu, cspn3d_wide.cu)
enum class Family {
    Normalised,   // weights gathered from the neighbours' guidance and normalised; 2D K in {5, 7}, 3D K = 5 with `mode`
                  // (2D and 3D backward: K = 3 too)
    Paddle,       // 2D 'paddle' own-location norm, K in {3, 5, 7} (in 3D it is mode 2 of Normalised)
    Gates,        // caller-supplied gates used as given; 2D K in {3, 5, 7}, 3D K in {3, 5}
};

// 2D.  Paddle and Gates: p.sparse null, p.gch == K*K-1, p.guidance [B][K*K-1][H][W].  fan non-null: the fused gather
// keep (Normalised, p.keep): one more B*C*H*W plane in either workspace; grad_sparse as in bwd2d
size_t widek_workspace_bytes(int B, int C, int H, int W, int K, int iters, Family family, bool keep = false);
int widek_forward(const Problem2D& p, int K, Family family, void* ws, size_t ws_bytes, cudaStream_t stream, int* launches,
                  const Fan* fan = nullptr);
size_t widek_bwd_workspace_bytes(int B, int C, int H, int W, int K, int iters, Family family, bool keep = false);
int widek_backward(const Problem2D& p, int K, Family family, const float* grad_out, float* grad_guidance, float* grad_blur,
                   void* ws, size_t ws_bytes, cudaStream_t stream, int* launches, float* grad_sparse = nullptr);

// 2D aggregation of the normalised family (DESIGN.md section 4.20): out = sum_j step_weight[j] * d_{steps[j]}, p.iters =
// steps[n_steps-1]; p.keep as above.  grad_* may be null
size_t aggregate2d_workspace_bytes(int B, int C, int H, int W, int K, bool keep);
size_t aggregate2d_bwd_workspace_bytes(int B, int C, int H, int W, int K, int N, bool keep);
int aggregate2d_forward(const Problem2D& p, int K, const float* step_weight, const int* steps, int n_steps, void* ws,
                        size_t ws_bytes, cudaStream_t stream, int* launches);
int aggregate2d_backward(const Problem2D& p, int K, const float* step_weight, const int* steps, int n_steps, const float* grad_out,
                         float* grad_guidance, float* grad_blur, float* grad_sparse, float* grad_step_weight, void* ws,
                         size_t ws_bytes, cudaStream_t stream, int* launches);

// volumes per launch group of the 3D paths: `planes` workspace planes per volume (27 for 3x3x3, K^3 for K x K x K)
int group3d(int B, int C, int D, int H, int W, int iters, int planes);
size_t generic3d_workspace_bytes(int B, int C, int D, int H, int W, int iters);
// fan non-null: the fused gather (cspn3d_fwd_gather_f32), destinations addressed like out
int generic3d_forward(const float* guidance, const float* feat, float* out, int B, int C, int D, int H, int W,
                      int iters, int mode, void* ws, size_t ws_bytes, cudaStream_t stream, int* launches,
                      const Fan* fan = nullptr);

// 3D, Normalised (guidance [B][K^3-1][D][H][W], mode 0 signed / 1 abs / 2 'paddle') or Gates (gates of that shape, mode
// unused).  fan non-null: the fused gather.  The normalised forward is K = 5 only (K = 3: generic3d_forward)
size_t widek3d_workspace_bytes(int B, int C, int D, int H, int W, int K, int iters, Family family);
int widek3d_forward(const float* guidance, const float* feat, float* out, int B, int C, int D, int H, int W, int K, int iters,
                    Family family, int mode, void* ws, size_t ws_bytes, cudaStream_t stream, int* launches,
                    const Fan* fan = nullptr);
size_t widek3d_bwd_workspace_bytes(int C, int D, int H, int W, int K, int iters, Family family);
int widek3d_backward(const float* guidance, const float* feat, const float* grad_out, float* grad_g, float* grad_feat, int B, int C,
                     int D, int H, int W, int K, int iters, Family family, int mode, void* ws, size_t ws_bytes,
                     cudaStream_t stream, int* launches);

// Unpool + crop + 3x3 convolution of the guidance / depth heads (unpool_conv.cu); shapes checked by the caller
int unpool_conv_launchable(int B, int Cin, int Cout, const char** why);
size_t unpool_conv_bwd_workspace_bytes(int B, int Cin, int H, int W, int Cout);
int unpool_conv_forward(const float* x, const float* w, float* out, int B, int Cin, int h, int wd, int Cout, int H, int W,
                        cudaStream_t st, int* launches);
int unpool_conv_backward(const float* x, const float* w, const float* g, float* gx, float* gw, int B, int Cin, int h, int wd,
                         int Cout, int H, int W, void* ws, cudaStream_t st, int* launches);

// Trilinear resampling, the Paddle module's resize_trilinear (resize_trilinear.cu); arguments checked by the caller.
// slices = B*C; (D, H, W) the input's size and (Do, Ho, Wo) the output's
int resize_trilinear_launchable(int D, int H, int W, int Do, int Ho, int Wo, const char** why);
size_t resize_trilinear_bwd_workspace_bytes(int D, int H, int W, int Do, int Ho, int Wo);
int resize_trilinear_forward(const float* x, float* out, long long slices, int D, int H, int W, int Do, int Ho, int Wo,
                             int align_corners, int align_mode, cudaStream_t st, int* launches);
int resize_trilinear_backward(const float* grad_out, float* grad_x, long long slices, int D, int H, int W, int Do, int Ho,
                              int Wo, int align_corners, int align_mode, void* ws, cudaStream_t st, int* launches);

// Disparity regression from a low-resolution cost volume (disparity_regression.cu): resize_trilinear to (Do, Ho, Wo), softmax
// over Do and the expectation; arguments checked by the caller (resize's checks, then launchable).  The backward's workspace
// is resize's tables, resize_trilinear_bwd_workspace_bytes()
int disparity_regression_launchable(int D, int H, int W, int Do, int Ho, int Wo, int align_corners, int align_mode,
                                    const char** why);
int disparity_regression_forward(const float* cost, float* out, long long slices, int D, int H, int W, int Do, int Ho, int Wo,
                                 int align_corners, int align_mode, cudaStream_t st, int* launches);
int disparity_regression_backward(const float* cost, const float* grad_out, float* grad_cost, long long slices, int D, int H,
                                  int W, int Do, int Ho, int Wo, int align_corners, int align_mode, void* ws, cudaStream_t st,
                                  int* launches);

// Stereo cost volumes from left and right feature maps (cost_volume.cu): the concatenation volume (G == 0) and the
// group-wise correlation volume; arguments checked by the caller (sizes, F % G, pointers, then launchable)
int cost_volume_launchable(int F, int H, int W, int D, int G, const char** why);
int concat_volume_forward(const float* left, const float* right, float* out, int B, int F, int H, int W, int D,
                          cudaStream_t st, int* launches);
int concat_volume_backward(const float* grad_out, float* grad_left, float* grad_right, int B, int F, int H, int W, int D,
                           cudaStream_t st, int* launches);
int gwc_volume_forward(const float* left, const float* right, float* out, int B, int F, int H, int W, int D, int G,
                       cudaStream_t st, int* launches);
int gwc_volume_backward(const float* left, const float* right, const float* grad_out, float* grad_left, float* grad_right,
                        int B, int F, int H, int W, int D, int G, cudaStream_t st, int* launches);

// Affinity pooling, the CSPN stereo network's spatial pyramid pooling (affinity_pool.cu): L <= 8 levels of feat (B, C, H, W)
// pooled with the gates (B, L, H, W) into one level-major buffer; arguments checked by the caller (sizes, kernel sizes,
// pointers, then launchable)
constexpr int kAffinityPoolMaxLevels = 8;
int affinity_pool_launchable(int B, int C, int H, int W, int L, const int* kernel_sizes, const char** why);
int affinity_pool_forward(const float* feat, const float* gate, float* out, int B, int C, int H, int W, int L,
                          const int* kernel_sizes, cudaStream_t st, int* launches);
int affinity_pool_backward(const float* feat, const float* gate, const float* out, const float* grad_out, float* grad_feat,
                           float* grad_gate, int B, int C, int H, int W, int L, const int* kernel_sizes, cudaStream_t st,
                           int* launches);

// Affinity fusion, the CSPN stereo network's spatial pyramid fusion (affinity_fuse.cu): L <= 8 levels (B, C, h_l, w_l),
// level_hw = (h_0, w_0, h_1, w_1, ...), resampled to (H, W) and combined with the normalised gates (B, L, H, W); arguments
// checked by the caller (sizes, flags, pointers, then launchable).  The backward's workspace holds the weight planes and the
// row pass, affinity_fuse_bwd_workspace_bytes() (0 when it would reach 2^62 bytes)
constexpr int kAffinityFuseMaxLevels = 8;
int affinity_fuse_launchable(int B, int C, int H, int W, int L, const int* level_hw, const char** why);
size_t affinity_fuse_bwd_workspace_bytes(int B, int C, int H, int W, int L, const int* level_hw);
int affinity_fuse_forward(const float* const* levels, const int* level_hw, const float* gate, float* out, int B, int C, int H,
                          int W, int L, int align_corners, int align_mode, cudaStream_t st, int* launches);
int affinity_fuse_backward(const float* const* levels, const int* level_hw, const float* gate, const float* out,
                           const float* grad_out, float* const* grad_levels, float* grad_gate, int B, int C, int H, int W, int L,
                           int align_corners, int align_mode, void* ws, cudaStream_t st, int* launches);

// Atrous affinity pooling, the CSPN stereo network's ACSPP (affinity_atrous.cu): L <= 8 levels of feat (B, C, H, W), level l
// a 3 x 3 CSPN step dilated by dilations[l] with the gates (B, 9L, H, W), into out (B, L*C, H, W); arguments checked by the
// caller (sizes, rates, pointers, then launchable).  The backward's workspace holds the weight planes (B, 9L, H, W),
// affinity_atrous_bwd_workspace_bytes() (0 when it would reach 2^60 bytes)
constexpr int kAffinityAtrousMaxLevels = 8;
int affinity_atrous_launchable(int B, int C, int H, int W, int L, const char** why);
size_t affinity_atrous_bwd_workspace_bytes(int B, int H, int W, int L);
int affinity_atrous_forward(const float* feat, const float* gate, float* out, int B, int C, int H, int W, int L,
                            const int* dilations, cudaStream_t st, int* launches);
int affinity_atrous_backward(const float* feat, const float* gate, const float* out, const float* grad_out, float* grad_feat,
                             float* grad_gate, int B, int C, int H, int W, int L, const int* dilations, void* ws, cudaStream_t st,
                             int* launches);

// Non-local 2D propagation, NLSPN's (cspn2d_nonlocal.cu): K in {3, 5, 7}, N steps of feat (B, C, H, W) with the learned
// offsets (B, 2T, H, W) and affinities (B, T, H, W), sparse (B, C, H, W) or nullptr; arguments checked by the caller (sizes,
// pointers, then launchable).  The forward's workspace is the h~ ping-pong; the backward's also holds every h~_t and
// lambda~_t, the transposed index and the radix sort's scratch (0 when the sort cannot be sized)
int nonlocal2d_launchable(int B, int C, int H, int W, int K, const char** why);
size_t nonlocal2d_workspace_bytes(int B, int C, int H, int W, int N);
size_t nonlocal2d_bwd_workspace_bytes(int B, int C, int H, int W, int K, int N);
int nonlocal2d_forward(const float* feat, const float* offset, const float* affinity, const float* sparse, float* out, int B, int C,
                       int H, int W, int K, int N, void* ws, cudaStream_t st, int* launches);
int nonlocal2d_backward(const float* feat, const float* offset, const float* affinity, const float* sparse, const float* grad_out,
                        float* grad_feat, float* grad_offset, float* grad_affinity, float* grad_sparse, int B, int C, int H, int W,
                        int K, int N, void* ws, cudaStream_t st, int* launches);

// Dilated K x K propagation with a centre weight on d_0 and a learned confidence, PENet's DA-CSPN++ (cspn2d_dilated.cu):
// K in {3, 5, 7}, dilation in [1, 4], N steps of blur (B, C, H, W) with kernel (B, K*K, H, W); sparse and conf (B, 1, H, W)
// or both nullptr; arguments checked by the caller (sizes, pointers, then launchable).  The forward's workspace is the
// ping-pong buffer; the backward's holds lambda_0 .. lambda_{N-1} and d_1 .. d_{N-1}
int dilated2d_launchable(int B, int C, int H, int W, const char** why);
size_t dilated2d_workspace_bytes(int B, int C, int H, int W, int N);
size_t dilated2d_bwd_workspace_bytes(int B, int C, int H, int W, int N);
int dilated2d_forward(const float* kern, const float* blur, const float* sparse, const float* conf, float* out, int B, int C, int H,
                      int W, int K, int dil, int N, void* ws, cudaStream_t st, int* launches);
int dilated2d_backward(const float* kern, const float* blur, const float* sparse, const float* conf, const float* grad_out,
                       float* grad_kern, float* grad_blur, float* grad_sparse, float* grad_conf, int B, int C, int H, int W, int K,
                       int dil, int N, void* ws, cudaStream_t st, int* launches);

// Dynamic K x K propagation with per-step ring attention and an anchor to d_0, DySPN's step (cspn2d_dynamic.cu): K in
// {3, 5, 7}, N steps of blur (B, C, H, W) with affinity (B, K*K, H, W) and attention (B, N*(K+1)/2, H, W); sparse and conf
// (B, 1, H, W) or both nullptr; arguments checked by the caller (sizes, pointers, then launchable).  The forward's
// workspace is the ping-pong buffer; the backward's holds lambda_0 .. lambda_{N-1} and d_1 .. d_{N-1}
int dynamic2d_launchable(int B, int C, int H, int W, const char** why);
size_t dynamic2d_workspace_bytes(int B, int C, int H, int W, int N);
size_t dynamic2d_bwd_workspace_bytes(int B, int C, int H, int W, int N);
int dynamic2d_forward(const float* aff, const float* att, const float* blur, const float* sparse, const float* conf, float* out, int B,
                      int C, int H, int W, int K, int N, void* ws, cudaStream_t st, int* launches);
int dynamic2d_backward(const float* aff, const float* att, const float* blur, const float* sparse, const float* conf,
                       const float* grad_out, float* grad_aff, float* grad_att, float* grad_blur, float* grad_sparse, float* grad_conf,
                       int B, int C, int H, int W, int K, int N, void* ws, cudaStream_t st, int* launches);

// Linear three-way scans, SPN's propagation (cspn2d_linear.cu): feat (B, C, H, W), gate (B, 3*nd*Cg, H, W) with Cg 1 or C,
// mask bits 1 l2r, 2 r2l, 4 t2b, 8 b2t; arguments checked by the caller (sizes, pointers, then launchable).  planes
// (nd, B, C, H, W) receive every direction's h when nd > 1 (the forward then merges them into out); with nd = 1 h goes to
// out, and the backward's planes are that output.  The backward's workspace holds grad_x's per-direction planes and the
// d* bytes (nd > 1) and a shared gate's per-channel gradient (Cg = 1 < C)
int linear2d_launchable(int B, int C, int H, int W, int mask, const char** why);
size_t linear2d_workspace_bytes(int B, int C, int H, int W, int mask);
size_t linear2d_bwd_workspace_bytes(int B, int C, int H, int W, int mask, int Cg);
int linear2d_forward(const float* feat, const float* gate, float* out, float* planes, int B, int C, int H, int W, int mask, int Cg,
                     cudaStream_t st, int* launches);
int linear2d_backward(const float* feat, const float* gate, const float* planes, const float* grad_out, float* grad_feat,
                      float* grad_gate, int B, int C, int H, int W, int mask, int Cg, void* ws, cudaStream_t st, int* launches);

}  // namespace cspn
