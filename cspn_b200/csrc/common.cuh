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

bool cluster2d_supported(const Problem2D& p, char* why, int why_len);
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

size_t generic3d_workspace_bytes(int B, int C, int D, int H, int W, int iters);
int generic3d_forward(const float* guidance, const float* feat, float* out, int B, int C, int D, int H, int W,
                      int iters, int mode, void* ws, size_t ws_bytes, cudaStream_t stream, int* launches);

size_t bwd3d_workspace_bytes(int C, int D, int H, int W, int iters);
int bwd3d(const float* guidance, const float* feat, const float* grad_out, float* grad_guidance, float* grad_feat, int B, int C,
          int D, int H, int W, int iters, int mode, void* ws, size_t ws_bytes, cudaStream_t stream, int* launches);

}  // namespace cspn
