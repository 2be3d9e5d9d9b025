// Atrous affinity pooling, the CSPN stereo network's ACSPP: L levels of one feature map feat (B, C, H, W), level l one CSPN
// step at stride 1 over the 3 x 3 neighbourhood dilated by r = r_l, with learned affinities gate (B, 9L, H, W), channel
// 9l + t the tap t = 3 (dy + 1) + (dx + 1) of level l, shared by all C channels.  At pixel p, every operation rounded on its
// own (no FMA contraction), every sum from its first term:
//
//   a_t = |gate[b, 9l + t, p]|,  S = sum_t a_t,  w_t = a_t / S,  out[b, lC + c, p] = sum_t w_t * f_c(p + r (dy_t, dx_t))
//
// with f = +0.0 outside the image (a tap that reads the padding still counts in S) and both sums in ascending t.  Backward
// (DESIGN.md section 4.19):
//   grad_gate[9l + t, p] = (T / S) * sgn(gate),  T = sum_c grad_out_l[c, p] * (f_c(p + r d_t) - out_l[c, p]), ascending c
//   grad_feat[c, q]      = sum over l ascending, then t ascending, of w_{l,t}(q - r_l d_t) * grad_out_l[c, q - r_l d_t],
//                          over the terms whose source pixel lies in the image (the centre tap always does)
// The bits depend on the arguments only: not on the launch, the stream, the batch split or the other levels of the call.
//
// Kernels, a thread per pixel along x (every tap's load is then a shifted, coalesced row), 1-D grids:
//   forward   one launch for every level: a thread forms its pixel's 9 weights once and walks a chunk of kFwdCh channels;
//   backward  1. a thread per (b, l, pixel) recomputes S and w with the forward's bits, writes the w planes (B, 9L, H, W) to
//                the workspace and grad_gate, walking all C channels for the 9 sums T;
//             2. a thread per (b, pixel) and kBwdCh channels gathers grad_feat from the w planes at the source pixels.
// No atomics, no memset; every output and workspace element is written once, and no workspace element is read before the
// first kernel has written it.
#include "common.cuh"

namespace cspn {
namespace {

constexpr int kThreads = 128;
constexpr int kFwdCh = 32;            // forward: channels per thread
constexpr int kBwdCh = 8;             // grad_feat gather: channels per thread

struct Rates {
    int r[kAffinityAtrousMaxLevels];
    int L;
};

__device__ __forceinline__ float sgn_of(float g) { return (float)(g > 0.f) - (float)(g < 0.f); }

// The 9 taps of pixel (y, x) at rate r: offsets into a plane and the mask of the taps inside the image
__device__ __forceinline__ unsigned tap_offsets(int y, int x, int r, int H, int W, int off[9]) {
    unsigned in = 0;
#pragma unroll
    for (int t = 0; t < 9; ++t) {
        const int yy = y + r * (t / 3 - 1), xx = x + r * (t % 3 - 1);
        const bool inside = yy >= 0 && yy < H && xx >= 0 && xx < W;
        off[t] = inside ? yy * W + xx : 0;
        in |= (unsigned)inside << t;
    }
    return in;
}

// S and the weights w_t = |g_t| / S of one level at one pixel; g points at tap 0's gate, taps a plane apart
__device__ __forceinline__ float level_weights(const float* __restrict__ g, size_t plane, float w[9]) {
#pragma unroll
    for (int t = 0; t < 9; ++t) w[t] = fabsf(__ldg(g + t * plane));
    float S = w[0];
#pragma unroll
    for (int t = 1; t < 9; ++t) S = __fadd_rn(S, w[t]);
#pragma unroll
    for (int t = 0; t < 9; ++t) w[t] = __fdiv_rn(w[t], S);
    return S;
}

// ---- forward: grid (B * L * channel chunks * H * x blocks) ------------------------------------------------------------------
__global__ void __launch_bounds__(kThreads)
affinity_atrous_fwd_kernel(const float* __restrict__ feat, const float* __restrict__ gate, float* __restrict__ out, int C, int H,
                           int W, int xblocks, int chunks, const __grid_constant__ Rates P) {
    long long e = blockIdx.x;
    const int x = (int)(e % xblocks) * kThreads + threadIdx.x;
    e /= xblocks;
    const int y = (int)(e % H);
    e /= H;
    const int cc = (int)(e % chunks);
    e /= chunks;
    const int l = (int)(e % P.L), b = (int)(e / P.L);
    if (x >= W) return;
    const size_t plane = (size_t)H * W;
    const int px = y * W + x;
    float w[9];
    level_weights(gate + ((size_t)b * 9 * P.L + 9 * l) * plane + px, plane, w);
    int off[9];
    const unsigned in = tap_offsets(y, x, P.r[l], H, W, off);
    const int c0 = cc * kFwdCh, nc = min(kFwdCh, C - c0);
    const float* f = feat + ((size_t)b * C + c0) * plane;
    float* o = out + (((size_t)b * P.L + l) * C + c0) * plane + px;
#pragma unroll 2
    for (int c = 0; c < nc; ++c) {
        float v[9];
#pragma unroll
        for (int t = 0; t < 9; ++t) v[t] = (in >> t & 1u) ? __ldg(f + off[t]) : 0.f;
        float acc = __fmul_rn(w[0], v[0]);
#pragma unroll
        for (int t = 1; t < 9; ++t) acc = __fadd_rn(acc, __fmul_rn(w[t], v[t]));
        o[(size_t)c * plane] = acc;
        f += plane;
    }
}

// ---- backward 1: grid (B * L * H * x blocks); grad_gate and the w planes -------------------------------------------------------
__global__ void __launch_bounds__(kThreads)
affinity_atrous_gate_kernel(const float* __restrict__ feat, const float* __restrict__ gate, const float* __restrict__ out,
                            const float* __restrict__ gout, float* __restrict__ ggate, float* __restrict__ wpl, int C, int H,
                            int W, int xblocks, const __grid_constant__ Rates P) {
    long long e = blockIdx.x;
    const int x = (int)(e % xblocks) * kThreads + threadIdx.x;
    e /= xblocks;
    const int y = (int)(e % H);
    e /= H;
    const int l = (int)(e % P.L), b = (int)(e / P.L);
    if (x >= W) return;
    const size_t plane = (size_t)H * W;
    const int px = y * W + x;
    const size_t g0 = ((size_t)b * 9 * P.L + 9 * l) * plane + px;   // tap 0 of the level in gate, grad_gate and the w planes
    float w[9];
    const float S = level_weights(gate + g0, plane, w);
#pragma unroll
    for (int t = 0; t < 9; ++t) wpl[g0 + t * plane] = w[t];
    int off[9];
    const unsigned in = tap_offsets(y, x, P.r[l], H, W, off);
    const float* f = feat + (size_t)b * C * plane;
    const size_t o0 = ((size_t)b * P.L + l) * C * plane + px;
    float T[9];
#pragma unroll 1
    for (int c = 0; c < C; ++c) {
        const float go = __ldg(gout + o0 + (size_t)c * plane), o = __ldg(out + o0 + (size_t)c * plane);
#pragma unroll
        for (int t = 0; t < 9; ++t) {
            const float v = (in >> t & 1u) ? __ldg(f + off[t]) : 0.f;
            const float pr = __fmul_rn(go, __fsub_rn(v, o));
            T[t] = c == 0 ? pr : __fadd_rn(T[t], pr);
        }
        f += plane;
    }
#pragma unroll
    for (int t = 0; t < 9; ++t) ggate[g0 + t * plane] = __fmul_rn(__fdiv_rn(T[t], S), sgn_of(__ldg(gate + g0 + t * plane)));
}

// ---- backward 2: grid (B * channel chunks * H * x blocks); grad_feat gathered from the w planes --------------------------------
__global__ void __launch_bounds__(kThreads)
affinity_atrous_feat_kernel(const float* __restrict__ gout, const float* __restrict__ wpl, float* __restrict__ gfeat, int C,
                            int H, int W, int xblocks, int chunks, const __grid_constant__ Rates P) {
    long long e = blockIdx.x;
    const int x = (int)(e % xblocks) * kThreads + threadIdx.x;
    e /= xblocks;
    const int y = (int)(e % H);
    e /= H;
    const int cc = (int)(e % chunks), b = (int)(e / chunks);
    if (x >= W) return;
    const size_t plane = (size_t)H * W;
    const int c0 = cc * kBwdCh, nc = min(kBwdCh, C - c0);
    float acc[kBwdCh];
    bool first = true;
#pragma unroll 1
    for (int l = 0; l < P.L; ++l) {
        const int r = P.r[l];
        const float* wl = wpl + ((size_t)b * 9 * P.L + 9 * l) * plane;
        const float* gl = gout + (((size_t)b * P.L + l) * C + c0) * plane;
#pragma unroll
        for (int t = 0; t < 9; ++t) {
            const int sy = y - r * (t / 3 - 1), sx = x - r * (t % 3 - 1);        // the pixel whose tap t reads (y, x)
            if (sy < 0 || sy >= H || sx < 0 || sx >= W) continue;
            const int sp = sy * W + sx;
            const float wt = __ldg(wl + t * plane + sp);
#pragma unroll
            for (int k = 0; k < kBwdCh; ++k) {
                if (k >= nc) break;
                const float term = __fmul_rn(wt, __ldg(gl + (size_t)k * plane + sp));
                acc[k] = first ? term : __fadd_rn(acc[k], term);
            }
            first = false;
        }
    }
    float* gf = gfeat + ((size_t)b * C + c0) * plane + (size_t)y * W + x;
#pragma unroll
    for (int k = 0; k < kBwdCh; ++k)
        if (k < nc) gf[(size_t)k * plane] = acc[k];
}

Rates make_rates(int L, const int* dilations) {
    Rates P{};
    P.L = L;
    for (int l = 0; l < L; ++l) P.r[l] = dilations[l];
    return P;
}

long long ceil_div(long long a, long long b) { return (a + b - 1) / b; }

// The three grids, in blocks
struct Grids {
    long long fwd, gate, feat;
};

Grids grids(int B, int C, int H, int W, int L) {
    const long long rows = (long long)H * ceil_div(W, kThreads);
    return {(long long)B * L * ceil_div(C, kFwdCh) * rows, (long long)B * L * rows, (long long)B * ceil_div(C, kBwdCh) * rows};
}

}  // namespace

size_t affinity_atrous_bwd_workspace_bytes(int B, int H, int W, int L) {
    const long long n = (long long)B * 9 * L;                               // < 2^38
    const long long hw = (long long)H * W;
    return hw > ((1ll << 60) / 4) / n ? 0 : (size_t)(n * hw) * sizeof(float);
}

int affinity_atrous_launchable(int B, int C, int H, int W, int L, const char** why) {
    if ((long long)H * W >= (1ll << 31)) { *why = "a (B, channel) slice has >= 2^31 elements"; return 0; }
    const Grids g = grids(B, C, H, W, L);
    if (g.fwd >= (1ll << 31)) { *why = "the forward grid has >= 2^31 blocks"; return 0; }
    if (g.gate >= (1ll << 31) || g.feat >= (1ll << 31)) { *why = "a backward grid has >= 2^31 blocks"; return 0; }
    if (affinity_atrous_bwd_workspace_bytes(B, H, W, L) == 0) { *why = "the backward's workspace is >= 2^60 bytes"; return 0; }
    return 1;
}

int affinity_atrous_forward(const float* feat, const float* gate, float* out, int B, int C, int H, int W, int L,
                            const int* dilations, cudaStream_t st, int* launches) {
    const Rates P = make_rates(L, dilations);
    const Grids g = grids(B, C, H, W, L);
    affinity_atrous_fwd_kernel<<<(unsigned)g.fwd, kThreads, 0, st>>>(feat, gate, out, C, H, W, (int)ceil_div(W, kThreads),
                                                                     (int)ceil_div(C, kFwdCh), P);
    CSPN_CUDA_TRY(cudaGetLastError());
    *launches = 1;
    return CSPN_OK;
}

int affinity_atrous_backward(const float* feat, const float* gate, const float* out, const float* grad_out, float* grad_feat,
                             float* grad_gate, int B, int C, int H, int W, int L, const int* dilations, void* ws, cudaStream_t st,
                             int* launches) {
    const Rates P = make_rates(L, dilations);
    const Grids g = grids(B, C, H, W, L);
    const int xblocks = (int)ceil_div(W, kThreads);
    float* wpl = static_cast<float*>(ws);
    affinity_atrous_gate_kernel<<<(unsigned)g.gate, kThreads, 0, st>>>(feat, gate, out, grad_out, grad_gate, wpl, C, H, W, xblocks,
                                                                       P);
    CSPN_CUDA_TRY(cudaGetLastError());
    affinity_atrous_feat_kernel<<<(unsigned)g.feat, kThreads, 0, st>>>(grad_out, wpl, grad_feat, C, H, W, xblocks,
                                                                       (int)ceil_div(C, kBwdCh), P);
    CSPN_CUDA_TRY(cudaGetLastError());
    *launches = 2;
    return CSPN_OK;
}

}  // namespace cspn
