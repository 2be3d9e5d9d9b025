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

// ---- problem descriptors --------------------------------------------------------------------
struct Problem2D {
    const float* guidance;  // [B][gch][H][W]
    const float* blur;      // [B][C][H][W]
    const float* sparse;    // [B][1][H][W] or nullptr
    float* out;             // [B][C][H][W]
    int B, C, H, W, gch, iters, norm_abs;
};

// ---- per-algorithm launchers (each returns a cspn_status; enqueue only, no sync) -------------
size_t generic2d_workspace_bytes(int B, int C, int H, int W, int iters);
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

void launch_prep2d(const float* guidance, const float* sparse, float* wk, int B, int H, int W, int gch, int norm_abs,
                   cudaStream_t stream);
void launch_step2d(const float* wk, const float* d0, const float* cur, float* dst, int B, int C, int H, int W,
                   cudaStream_t stream);

size_t bwd2d_workspace_bytes(int B, int C, int H, int W, int iters);
int bwd2d(const Problem2D& p, const float* grad_out, float* grad_guidance, float* grad_blur, void* ws,
          size_t ws_bytes, cudaStream_t stream, int* launches);

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

// The FAN epilogue of the 3D step kernels: v, just stored at element o of dst, also to element o of every destination
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

// K x K kernels, K in {5, 7} (cspn2d_wide.cu); fan non-null: the fused gather
size_t widek_workspace_bytes(int B, int C, int H, int W, int K, int iters);
int widek_forward(const Problem2D& p, int K, void* ws, size_t ws_bytes, cudaStream_t stream, int* launches,
                  const Fan* fan = nullptr);
size_t widek_bwd_workspace_bytes(int B, int C, int H, int W, int K, int iters);
int widek_backward(const Problem2D& p, int K, const float* grad_out, float* grad_guidance, float* grad_blur, void* ws,
                   size_t ws_bytes, cudaStream_t stream, int* launches);
// 'paddle' own-location norm, K in {3, 5, 7}, on the same kernels and workspaces (p.sparse null, p.gch == K*K-1)
int widek_paddle_forward(const Problem2D& p, int K, void* ws, size_t ws_bytes, cudaStream_t stream, int* launches,
                         const Fan* fan = nullptr);
int widek_paddle_backward(const Problem2D& p, int K, const float* grad_out, float* grad_guidance, float* grad_blur, void* ws,
                          size_t ws_bytes, cudaStream_t stream, int* launches);
// caller-supplied gates, K in {3, 5, 7}: p.guidance [B][K*K-1][H][W] used as given (p.sparse null, p.gch == K*K-1)
size_t widek_gates_workspace_bytes(int B, int C, int H, int W, int iters);
size_t widek_gates_bwd_workspace_bytes(int B, int C, int H, int W, int iters);
int widek_gates_forward(const Problem2D& p, int K, void* ws, size_t ws_bytes, cudaStream_t stream, int* launches,
                        const Fan* fan = nullptr);
int widek_gates_backward(const Problem2D& p, int K, const float* grad_out, float* grad_gates, float* grad_feat, void* ws,
                         size_t ws_bytes, cudaStream_t stream, int* launches);

// volumes per launch group of the 3D paths: `planes` workspace planes per volume (27 for 3x3x3, K^3 for K x K x K)
int group3d(int B, int C, int D, int H, int W, int iters, int planes);
size_t generic3d_workspace_bytes(int B, int C, int D, int H, int W, int iters);
// fan non-null: the fused gather (cspn3d_fwd_gather_f32), destinations addressed like out
int generic3d_forward(const float* guidance, const float* feat, float* out, int B, int C, int D, int H, int W,
                      int iters, int mode, void* ws, size_t ws_bytes, cudaStream_t stream, int* launches,
                      const Fan* fan = nullptr);

size_t bwd3d_workspace_bytes(int C, int D, int H, int W, int iters);
int bwd3d(const float* guidance, const float* feat, const float* grad_out, float* grad_guidance, float* grad_feat, int B, int C,
          int D, int H, int W, int iters, int mode, void* ws, size_t ws_bytes, cudaStream_t stream, int* launches);

// K x K x K kernels, K = 5 (cspn3d_wide.cu); fan non-null: the fused gather
size_t widek3d_workspace_bytes(int B, int C, int D, int H, int W, int K, int iters);
int widek3d_forward(const float* guidance, const float* feat, float* out, int B, int C, int D, int H, int W, int K, int iters,
                    int mode, void* ws, size_t ws_bytes, cudaStream_t stream, int* launches, const Fan* fan = nullptr);
size_t widek3d_bwd_workspace_bytes(int C, int D, int H, int W, int K, int iters);
int widek3d_backward(const float* guidance, const float* feat, const float* grad_out, float* grad_g, float* grad_feat, int B, int C,
                     int D, int H, int W, int K, int iters, int mode, void* ws, size_t ws_bytes, cudaStream_t stream,
                     int* launches);
// caller-supplied gates [B][K^3-1][D][H][W], K in {3, 5} (cspn3d_wide.cu)
size_t widek3d_gates_workspace_bytes(int B, int C, int D, int H, int W, int iters);
size_t widek3d_gates_bwd_workspace_bytes(int C, int D, int H, int W, int iters);
int widek3d_gates_forward(const float* gates, const float* feat, float* out, int B, int C, int D, int H, int W, int K, int iters,
                          void* ws, size_t ws_bytes, cudaStream_t stream, int* launches, const Fan* fan = nullptr);
int widek3d_gates_backward(const float* gates, const float* feat, const float* grad_out, float* grad_g, float* grad_feat, int B,
                           int C, int D, int H, int W, int K, int iters, void* ws, size_t ws_bytes, cudaStream_t stream,
                           int* launches);

// Unpool + crop + 3x3 convolution of the guidance / depth heads (unpool_conv.cu); shapes checked by the caller
int unpool_conv_launchable(int B, int Cin, int Cout, const char** why);
size_t unpool_conv_bwd_workspace_bytes(int B, int Cin, int H, int W, int Cout);
int unpool_conv_forward(const float* x, const float* w, float* out, int B, int Cin, int h, int wd, int Cout, int H, int W,
                        cudaStream_t st, int* launches);
int unpool_conv_backward(const float* x, const float* w, const float* g, float* gx, float* gw, int B, int Cin, int h, int wd,
                         int Cout, int H, int W, void* ws, cudaStream_t st, int* launches);

}  // namespace cspn
