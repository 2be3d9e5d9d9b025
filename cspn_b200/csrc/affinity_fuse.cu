// Affinity fusion, the CSPN stereo network's spatial pyramid fusion: L levels x_l (B, C, h_l, w_l) of a feature pyramid
// combined at every pixel of the output (B, C, H, W) with learned, normalised affinities gate (B, L, H, W), forward and a
// deterministic backward.  At pixel q, with every operation rounded on its own (no FMA contraction):
//
//   a_l = |gate[b, l, q]|,  S = sum_l a_l,  w_l = a_l / S,  out[b, c, q] = sum_l w_l * u_l[c](q)
//
// u_l is level l resampled bilinearly to (H, W) with resize_trilinear's per-axis rule (tap_of / make_axis of
// resize_taps.cuh, DESIGN.md section 4.14):
//   u = l0h*(l0w*x[h0,w0] + l1w*x[h0,w1]) + l1h*(l0w*x[h1,w0] + l1w*x[h1,w1]),  left to right, every product computed.
// S and out are summed in ascending l from the first term.  Backward (DESIGN.md section 4.18):
//   grad_gate_l(q)  = (t_l / S) * sgn(gate_l(q)),  t_l = sum_c grad_out[c](q) * (u_l[c](q) - out[c](q)), ascending c
//   grad_x_l        = sum_oh (sum_ow v * lw) * lh with v = w_l(q) * grad_out[c](q): section 4.14's gather, each sum from
//                     0 in ascending o over the outputs that read the index, both products (v*l0 first) where i1 == i0
// The bits depend on the arguments only: not on the launch, the stream, the batch split or the other levels of the call.
//
// Kernels.  The forward gives a thread four consecutive outputs of one row and four channels; it forms S and each level's
// taps and weights once for them and stores a float4 when W % 4 == 0 and out is aligned.  The backward runs three kernels:
//   1. a thread per pixel writes grad_gate and the weight planes w_l (B, L, H, W) to the workspace;
//   2. the row pass: a thread per (b, c, oh, j) of every level writes R_l = sum_ow v * lw to the workspace;
//   3. the column pass: a thread per level cell writes grad_x_l = sum_oh R_l * lh.
// The row pass splits the coarsest levels' long sums (a 1 x 2 level read by thousands of outputs) over H threads.  No
// atomics, no memset; every output element is written once, +0.0 where no output reads a cell.
#include "common.cuh"
#include "resize_taps.cuh"

namespace cspn {
namespace {

constexpr int kFuseThreads = 256;
constexpr int kFuseCh = 4;            // channels per forward thread

struct FuseLevel {
    const float* x;                   // (B, C, ah.n_in, aw.n_in)
    float* gx;                        // its gradient (backward)
    Axis ah, aw;                      // n_in -> H, n_in -> W
    long long rows0;                  // first row-pass item (and workspace float) of the level
    long long cells0;                 // first column-pass item of the level
};

struct FuseLevels {
    FuseLevel lv[kAffinityFuseMaxLevels];
    int L;
};

__device__ __forceinline__ float sgn_of(float g) { return (float)(g > 0.f) - (float)(g < 0.f); }

// The level of a grid-stride item: the last l with first(l) <= e
template <class First>
__device__ __forceinline__ int level_of(const FuseLevels& P, long long e, First first) {
    int l = 0;
    while (l + 1 < P.L && first(P.lv[l + 1]) <= e) ++l;
    return l;
}

// ---- forward: grid (row quads of an image, (b, channel chunk) slices) ------------------------------------------------------
__global__ void __launch_bounds__(kFuseThreads)
affinity_fuse_fwd_kernel(const float* __restrict__ gate, float* __restrict__ out, int C, int H, int W, int quads,
                         long long slices, int vec, const __grid_constant__ FuseLevels P) {
    const int q = blockIdx.x * kFuseThreads + threadIdx.x;
    if (q >= H * quads) return;
    const int oh = q / quads, ow0 = q % quads * 4, L = P.L;
    const int chunks = (C + kFuseCh - 1) / kFuseCh;
    const size_t plane = (size_t)H * W;
    int ow[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) ow[k] = min(ow0 + k, W - 1);
    for (long long s = blockIdx.y; s < slices; s += gridDim.y) {
        const int b = (int)(s / chunks), c0 = (int)(s % chunks) * kFuseCh;
        const float* g = gate + (size_t)b * L * plane + (size_t)oh * W;
        float S[4];
#pragma unroll
        for (int k = 0; k < 4; ++k) S[k] = fabsf(__ldg(g + ow[k]));
        for (int l = 1; l < L; ++l)
#pragma unroll
            for (int k = 0; k < 4; ++k) S[k] = __fadd_rn(S[k], fabsf(__ldg(g + l * plane + ow[k])));
        float acc[kFuseCh][4] = {};
        for (int l = 0; l < L; ++l) {
            const FuseLevel& v = P.lv[l];
            const int hn = v.ah.n_in, wn = v.aw.n_in;
            const Tap th = tap_of(v.ah, oh);
            const int h1 = th.i0 + (th.i0 < hn - 1);
            const float l0h = __fsub_rn(1.f, th.l1);
            int w0[4], w1[4];
            float l0w[4], l1w[4], w[4];
#pragma unroll
            for (int k = 0; k < 4; ++k) {
                const Tap tw = tap_of(v.aw, ow[k]);
                w0[k] = tw.i0;
                w1[k] = tw.i0 + (tw.i0 < wn - 1);
                l1w[k] = tw.l1;
                l0w[k] = __fsub_rn(1.f, tw.l1);
                w[k] = __fdiv_rn(fabsf(__ldg(g + l * plane + ow[k])), S[k]);
            }
            const size_t lp = (size_t)hn * wn;
            const float* r0 = v.x + ((size_t)b * C + c0) * lp + (size_t)th.i0 * wn;
            const float* r1 = v.x + ((size_t)b * C + c0) * lp + (size_t)h1 * wn;
#pragma unroll
            for (int j = 0; j < kFuseCh; ++j) {
                if (c0 + j >= C) break;
#pragma unroll
                for (int k = 0; k < 4; ++k) {
                    const float e0 = __fadd_rn(__fmul_rn(l0w[k], __ldg(r0 + j * lp + w0[k])), __fmul_rn(l1w[k], __ldg(r0 + j * lp + w1[k])));
                    const float e1 = __fadd_rn(__fmul_rn(l0w[k], __ldg(r1 + j * lp + w0[k])), __fmul_rn(l1w[k], __ldg(r1 + j * lp + w1[k])));
                    const float t = __fmul_rn(w[k], __fadd_rn(__fmul_rn(l0h, e0), __fmul_rn(th.l1, e1)));
                    acc[j][k] = l == 0 ? t : __fadd_rn(acc[j][k], t);
                }
            }
        }
#pragma unroll
        for (int j = 0; j < kFuseCh; ++j) {
            if (c0 + j >= C) break;
            float* o = out + ((size_t)b * C + c0 + j) * plane + (size_t)oh * W + ow0;
            if (vec) {
                *reinterpret_cast<float4*>(o) = make_float4(acc[j][0], acc[j][1], acc[j][2], acc[j][3]);
            } else {
#pragma unroll
                for (int k = 0; k < 4; ++k)
                    if (ow0 + k < W) o[k] = acc[j][k];
            }
        }
    }
}

// ---- backward 1: grid (pixels of an image, images); grad_gate and the weight planes -----------------------------------------
__global__ void __launch_bounds__(kFuseThreads)
affinity_fuse_gate_kernel(const float* __restrict__ gate, const float* __restrict__ out, const float* __restrict__ gout,
                          float* __restrict__ ggate, float* __restrict__ wpl, int B, int C, int H, int W,
                          const __grid_constant__ FuseLevels P) {
    const int px = blockIdx.x * kFuseThreads + threadIdx.x;
    if (px >= H * W) return;
    const int oh = px / W, ow = px % W, L = P.L;
    const size_t plane = (size_t)H * W;
    for (int b = blockIdx.y; b < B; b += gridDim.y) {
        const float* g = gate + (size_t)b * L * plane + px;
        float S = fabsf(__ldg(g));
        for (int l = 1; l < L; ++l) S = __fadd_rn(S, fabsf(__ldg(g + l * plane)));
        const float* o = out + (size_t)b * C * plane + px;
        const float* go = gout + (size_t)b * C * plane + px;
#pragma unroll 1
        for (int l = 0; l < L; ++l) {
            const FuseLevel& v = P.lv[l];
            const int hn = v.ah.n_in, wn = v.aw.n_in;
            const Tap th = tap_of(v.ah, oh), tw = tap_of(v.aw, ow);
            const int h1 = th.i0 + (th.i0 < hn - 1), w1 = tw.i0 + (tw.i0 < wn - 1);
            const float l0h = __fsub_rn(1.f, th.l1), l0w = __fsub_rn(1.f, tw.l1);
            const float gl = __ldg(g + l * plane);
            wpl[((size_t)b * L + l) * plane + px] = __fdiv_rn(fabsf(gl), S);
            const size_t lp = (size_t)hn * wn;
            const float* r0 = v.x + (size_t)b * C * lp + (size_t)th.i0 * wn;
            const float* r1 = v.x + (size_t)b * C * lp + (size_t)h1 * wn;
            float t = 0.f;
            for (int c = 0; c < C; ++c) {
                const size_t xo = (size_t)c * lp;
                const float e0 = __fadd_rn(__fmul_rn(l0w, __ldg(r0 + xo + tw.i0)), __fmul_rn(tw.l1, __ldg(r0 + xo + w1)));
                const float e1 = __fadd_rn(__fmul_rn(l0w, __ldg(r1 + xo + tw.i0)), __fmul_rn(tw.l1, __ldg(r1 + xo + w1)));
                const float u = __fadd_rn(__fmul_rn(l0h, e0), __fmul_rn(th.l1, e1));
                const float pr = __fmul_rn(__ldg(go + (size_t)c * plane), __fsub_rn(u, __ldg(o + (size_t)c * plane)));
                t = c == 0 ? pr : __fadd_rn(t, pr);
            }
            ggate[((size_t)b * L + l) * plane + px] = __fmul_rn(__fdiv_rn(t, S), sgn_of(gl));
        }
    }
}

// ---- backward 2, the row pass: grid-stride over (b, c, oh, j) of every level ----------------------------------------------------
// rows[rows0 + ((b*C + c)*H + oh)*w_l + j] = sum over the ow that read j, ascending, of (w_l * grad_out[c]) * lw
__global__ void __launch_bounds__(kFuseThreads)
affinity_fuse_rows_kernel(const float* __restrict__ gout, const float* __restrict__ wpl, float* __restrict__ rows, int C,
                          int H, int W, long long total, const __grid_constant__ FuseLevels P) {
    const size_t plane = (size_t)H * W;
    for (long long e = (long long)blockIdx.x * kFuseThreads + threadIdx.x; e < total; e += (long long)gridDim.x * kFuseThreads) {
        const int l = level_of(P, e, [](const FuseLevel& v) { return v.rows0; });
        const FuseLevel& v = P.lv[l];
        const int wn = v.aw.n_in;
        long long r = e - v.rows0;
        const int j = (int)(r % wn);
        r /= wn;
        const int oh = (int)(r % H);
        const long long bc = r / H;
        const int b = (int)(bc / C);
        const float* go = gout + (size_t)bc * plane + (size_t)oh * W;
        const float* w = wpl + ((size_t)b * P.L + l) * plane + (size_t)oh * W;
        const int ob = first_output(v.aw, j - 1), oe = first_output(v.aw, j + 1);
        float acc = 0.f;
        for (int o = ob; o < oe; ++o) acc = add_tap(acc, __fmul_rn(__ldg(w + o), __ldg(go + o)), tap_of(v.aw, o), j, wn);
        rows[e] = acc;
    }
}

// ---- backward 3, the column pass: grid-stride over the cells (b, c, i, j) of every level -------------------------------------------
__global__ void __launch_bounds__(kFuseThreads)
affinity_fuse_cols_kernel(const float* __restrict__ rows, int C, int H, long long total, const __grid_constant__ FuseLevels P) {
    for (long long e = (long long)blockIdx.x * kFuseThreads + threadIdx.x; e < total; e += (long long)gridDim.x * kFuseThreads) {
        const int l = level_of(P, e, [](const FuseLevel& v) { return v.cells0; });
        const FuseLevel& v = P.lv[l];
        const int hn = v.ah.n_in, wn = v.aw.n_in;
        const long long r = e - v.cells0;
        const int j = (int)(r % wn), i = (int)(r / wn % hn);
        const long long bc = r / wn / hn;
        const float* col = rows + v.rows0 + (size_t)bc * H * wn + j;
        const int ob = first_output(v.ah, i - 1), oe = first_output(v.ah, i + 1);
        float acc = 0.f;
        for (int o = ob; o < oe; ++o) acc = add_tap(acc, __ldg(col + (size_t)o * wn), tap_of(v.ah, o), i, hn);
        v.gx[r] = acc;
    }
}

// The levels' parameters; *rows and *cells are the row-pass and column-pass item counts
FuseLevels plan_fuse(const float* const* levels, float* const* grad_levels, const int* level_hw, int B, int C, int H, int W,
                     int L, int align_corners, int align_mode, long long* rows, long long* cells) {
    FuseLevels P{};
    P.L = L;
    long long nr = 0, nc = 0;
    for (int l = 0; l < L; ++l) {
        FuseLevel& v = P.lv[l];
        v.x = levels[l];
        v.gx = grad_levels ? grad_levels[l] : nullptr;
        v.ah = make_axis(level_hw[2 * l], H, align_corners, align_mode);
        v.aw = make_axis(level_hw[2 * l + 1], W, align_corners, align_mode);
        v.rows0 = nr;
        v.cells0 = nc;
        nr += (long long)B * C * H * level_hw[2 * l + 1];
        nc += (long long)B * C * level_hw[2 * l] * level_hw[2 * l + 1];
    }
    *rows = nr;
    *cells = nc;
    return P;
}

// a * b, or -1 past 2^62
long long mul_capped(long long a, long long b) { return a > 0 && b > (1ll << 62) / a ? -1 : a * b; }

unsigned stride_blocks(long long items) {
    const long long n = (items + kFuseThreads - 1) / kFuseThreads;
    return (unsigned)(n < (1ll << 20) ? n : (1ll << 20));
}

}  // namespace

int affinity_fuse_launchable(int B, int C, int H, int W, int L, const int* level_hw, const char** why) {
    if ((long long)H * W >= (1ll << 31)) { *why = "the output has >= 2^31 elements per (B, channel) slice"; return 0; }
    for (int l = 0; l < L; ++l)
        if ((long long)level_hw[2 * l] * level_hw[2 * l + 1] >= (1ll << 31)) {
            *why = "a level has >= 2^31 elements per (B, channel) slice";
            return 0;
        }
    if (affinity_fuse_bwd_workspace_bytes(B, C, H, W, L, level_hw) == 0) { *why = "the backward's workspace is >= 2^62 bytes"; return 0; }
    return 1;
}

size_t affinity_fuse_bwd_workspace_bytes(int B, int C, int H, int W, int L, const int* level_hw) {
    long long n = mul_capped(mul_capped(B, L), (long long)H * W);
    for (int l = 0; l < L && n >= 0; ++l) {
        const long long r = mul_capped(mul_capped((long long)B * C, H), level_hw[2 * l + 1]);
        n = r < 0 || n + r >= (1ll << 60) ? -1 : n + r;
    }
    return n < 0 ? 0 : (size_t)n * sizeof(float);
}

int affinity_fuse_forward(const float* const* levels, const int* level_hw, const float* gate, float* out, int B, int C, int H,
                          int W, int L, int align_corners, int align_mode, cudaStream_t st, int* launches) {
    long long nr, nc;
    const FuseLevels P = plan_fuse(levels, nullptr, level_hw, B, C, H, W, L, align_corners, align_mode, &nr, &nc);
    const int quads = (W + 3) / 4;
    const long long slices = (long long)B * ((C + kFuseCh - 1) / kFuseCh);
    const int vec = W % 4 == 0 && (reinterpret_cast<uintptr_t>(out) & 15) == 0;
    const dim3 grid((unsigned)(((long long)H * quads + kFuseThreads - 1) / kFuseThreads), slice_blocks(slices));
    affinity_fuse_fwd_kernel<<<grid, kFuseThreads, 0, st>>>(gate, out, C, H, W, quads, slices, vec, P);
    CSPN_CUDA_TRY(cudaGetLastError());
    *launches = 1;
    return CSPN_OK;
}

int affinity_fuse_backward(const float* const* levels, const int* level_hw, const float* gate, const float* out,
                           const float* grad_out, float* const* grad_levels, float* grad_gate, int B, int C, int H, int W, int L,
                           int align_corners, int align_mode, void* ws, cudaStream_t st, int* launches) {
    long long nr, nc;
    const FuseLevels P = plan_fuse(levels, grad_levels, level_hw, B, C, H, W, L, align_corners, align_mode, &nr, &nc);
    float* wpl = static_cast<float*>(ws);
    float* rows = wpl + (size_t)B * L * H * W;
    const dim3 grid((unsigned)(((long long)H * W + kFuseThreads - 1) / kFuseThreads), slice_blocks(B));
    affinity_fuse_gate_kernel<<<grid, kFuseThreads, 0, st>>>(gate, out, grad_out, grad_gate, wpl, B, C, H, W, P);
    CSPN_CUDA_TRY(cudaGetLastError());
    affinity_fuse_rows_kernel<<<stride_blocks(nr), kFuseThreads, 0, st>>>(grad_out, wpl, rows, C, H, W, nr, P);
    CSPN_CUDA_TRY(cudaGetLastError());
    affinity_fuse_cols_kernel<<<stride_blocks(nc), kFuseThreads, 0, st>>>(rows, C, H, nc, P);
    CSPN_CUDA_TRY(cudaGetLastError());
    *launches = 3;
    return CSPN_OK;
}

}  // namespace cspn
