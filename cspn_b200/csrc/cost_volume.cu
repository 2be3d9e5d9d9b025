// Stereo cost volumes from left and right feature maps (B, F, H, W), forward and a deterministic backward, one launch
// each: the concatenation volume of PSMNet and the group-wise correlation volume of GwcNet.  The matched pixel of
// left[..., x] at disparity d is right[..., x - d]; cells with x < d are +0.0 whatever the inputs hold.
//
//   concat:  out[b, c, d, y, x] = left[b, c, y, x],  out[b, F + c, d, y, x] = right[b, c, y, x - d]     (x >= d)
//   gwc:     out[b, g, d, y, x] = (sum_{c in group g} left[b, c, y, x] * right[b, c, y, x - d]) / n       (x >= d)
//
// Operation order, every operation rounded on its own (no FMA contraction), every sum from its first term:
//   gwc forward      p_c = L_c * R_c summed in ascending c within the group, then / n
//   concat backward  grad_left[c,y,x]  = sum_{d=0}^{min(x, D-1)} g[c, d, y, x]
//                    grad_right[c,y,x] = sum_{d=0}^{min(W-1-x, D-1)} g[F + c, d, y, x + d]          (ascending d)
//   gwc backward     t = g[grp, d, y, .] / n
//                    grad_left[c,y,x]  = sum_d t(x) * R[c, y, x - d],  grad_right[c,y,x] = sum_d t(x + d) * L[c, y, x + d]
//                    (ascending d, the ranges of the concat backward)
// The bits depend on the arguments only: not on the tile, the stream, the batch split or the run.
//
// Kernels.  The two forwards and the gwc backward own a tile of TX columns of one row y (and a chunk of channels or one
// group of one image); they stage the rows they read in shared memory, the shifted rows with their D - 1 halo clipped to
// [0, W).  Every output element is written once, zeros included: no memset, no atomics, no workspace.  The concat backward
// needs no staging: a thread per input element walks d, and the reads of g[..., x + d] are contiguous across a warp.
//
// Limits: the host halves TX from 128 until a tile fits two CTAs per SM; a shape whose 1-column tile does not fit in
// 227 KB is CSPN_ERR_UNSUPPORTED (DESIGN.md section 4.16 gives the D at which that happens).
#include <algorithm>

#include "common.cuh"

namespace cspn {
namespace {

constexpr int kThreads = 256;
constexpr size_t kSmemSoft = 110 * 1024;   // two CTAs per SM
constexpr size_t kSmemHard = 227 * 1024;   // the sm_90 per-CTA maximum
constexpr int kConcatChunk = 4;            // channels per CTA, concat forward
constexpr int kGwcBwdChunk = 8;            // channels per CTA, gwc backward
constexpr int kDisp = 8;                   // disparities per thread, gwc forward

unsigned slice_blocks(long long slices) { return (unsigned)(slices < 65535 ? slices : 65535); }

__device__ __forceinline__ size_t row_of(int b, int c, int y, int C, int H, int W) {
    return (((size_t)b * C + c) * H + y) * W;
}

// Stages n elements of rows src + row(c) into dst[c * pitch ...] for c < nc (the row of channel c is c * H * W further)
__device__ __forceinline__ void stage_rows(float* dst, int pitch, const float* src, size_t cstride, int nc, int n) {
    for (int e = threadIdx.x; e < nc * n; e += blockDim.x) {
        const int c = e / n, k = e % n;
        dst[c * pitch + k] = __ldg(src + (size_t)c * cstride + k);
    }
}

// ---- concat forward: grid (x tiles * H, B * channel chunks) ------------------------------------------------------------
// left row [x0, x0 + nx) as ls[c][TX], right row [r_lo, x0 + nx) as rs[c][RP]
__global__ void __launch_bounds__(kThreads)
concat_volume_fwd_kernel(const float* __restrict__ L, const float* __restrict__ R, float* __restrict__ out, int B, int F,
                         int H, int W, int D, int TX, int RP, int tiles_x, int vec) {
    extern __shared__ float4 smem4[];
    float* ls = reinterpret_cast<float*>(smem4);
    float* rs = ls + kConcatChunk * TX;
    const int y = (int)(blockIdx.x / tiles_x), x0 = (int)(blockIdx.x % tiles_x) * TX;
    const int nx = min(TX, W - x0), r_lo = max(x0 - D + 1, 0), nr = x0 + nx - r_lo;
    const int chunks = (F + kConcatChunk - 1) / kConcatChunk;
    const size_t plane = (size_t)H * W;
    for (long long s = blockIdx.y; s < (long long)B * chunks; s += gridDim.y) {
        const int b = (int)(s / chunks), c0 = (int)(s % chunks) * kConcatChunk, nc = min(kConcatChunk, F - c0);
        __syncthreads();                        // the last slice's reads are done
        stage_rows(ls, TX, L + row_of(b, c0, y, F, H, W) + x0, plane, nc, nx);
        stage_rows(rs, RP, R + row_of(b, c0, y, F, H, W) + r_lo, plane, nc, nr);
        __syncthreads();
        // rows (part, c, d) of the output, part 0 from left and 1 from right
        const int rows = 2 * nc * D;
        if (vec) {                              // nx and x0 are multiples of 4, and so is every row's start
            const int q = nx / 4;
            for (int it = threadIdx.x; it < rows * q; it += blockDim.x) {
                const int k = it % q, r = it / q, d = r % D, c = (r / D) % nc, part = r / (D * nc);
                const int x = x0 + 4 * k;
                float v[4];
#pragma unroll
                for (int j = 0; j < 4; ++j)
                    v[j] = x + j < d ? 0.f : part == 0 ? ls[c * TX + 4 * k + j] : rs[c * RP + x + j - d - r_lo];
                float* dst = out + (((size_t)b * 2 * F + part * F + c0 + c) * D + d) * plane + (size_t)y * W + x;
                *reinterpret_cast<float4*>(dst) = make_float4(v[0], v[1], v[2], v[3]);
            }
        } else {
            for (int it = threadIdx.x; it < rows * nx; it += blockDim.x) {
                const int k = it % nx, r = it / nx, d = r % D, c = (r / D) % nc, part = r / (D * nc);
                const int x = x0 + k;
                out[(((size_t)b * 2 * F + part * F + c0 + c) * D + d) * plane + (size_t)y * W + x] =
                    x < d ? 0.f : part == 0 ? ls[c * TX + k] : rs[c * RP + x - d - r_lo];
            }
        }
    }
}

// ---- concat backward: a thread per input element (b, c, y, x) -----------------------------------------------------------
__global__ void __launch_bounds__(kThreads)
concat_volume_bwd_kernel(const float* __restrict__ g, float* __restrict__ gl, float* __restrict__ gr, int B, int F, int H,
                         int W, int D) {
    const long long total = (long long)B * F * H * W;
    const size_t plane = (size_t)H * W;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const int x = (int)(i % W);
        const long long r = i / W;                          // (b * F + c) * H + y
        const long long bc = r / H;
        const int y = (int)(r % H), c = (int)(bc % F), b = (int)(bc / F);
        const float* gL = g + ((size_t)b * 2 * F + c) * D * plane + (size_t)y * W + x;
        const float* gR = gL + (size_t)F * D * plane;
        const int nl = min(x, D - 1), nr = min(W - 1 - x, D - 1);
        float a = gL[0];
#pragma unroll 4
        for (int d = 1; d <= nl; ++d) a = __fadd_rn(a, gL[(size_t)d * plane]);
        float s = gR[0];
#pragma unroll 4
        for (int d = 1; d <= nr; ++d) s = __fadd_rn(s, gR[(size_t)d * plane + d]);
        gl[i] = a;
        gr[i] = s;
    }
}

// ---- gwc forward: grid (x tiles * H, B * G); left rows of the group as ls[c][TX], right rows as rs[c][RP] ------------------
// A thread owns a column x and kDisp consecutive disparities, and keeps their sums in registers over the group's channels
__global__ void __launch_bounds__(kThreads)
gwc_volume_fwd_kernel(const float* __restrict__ L, const float* __restrict__ R, float* __restrict__ out, int B, int F, int H,
                      int W, int D, int G, int TX, int RP, int tiles_x) {
    extern __shared__ float4 smem4[];
    const int n = F / G;
    float* ls = reinterpret_cast<float*>(smem4);
    float* rs = ls + n * TX;
    const int y = (int)(blockIdx.x / tiles_x), x0 = (int)(blockIdx.x % tiles_x) * TX;
    const int nx = min(TX, W - x0), r_lo = max(x0 - D + 1, 0), nr = x0 + nx - r_lo;
    const int ndc = (min(D, x0 + nx) + kDisp - 1) / kDisp;   // planes d >= x0 + nx are zero in the whole tile
    const float fn = (float)n;
    const size_t plane = (size_t)H * W;
    for (long long s = blockIdx.y; s < (long long)B * G; s += gridDim.y) {
        const int b = (int)(s / G), grp = (int)(s % G);
        __syncthreads();
        stage_rows(ls, TX, L + row_of(b, grp * n, y, F, H, W) + x0, plane, n, nx);
        stage_rows(rs, RP, R + row_of(b, grp * n, y, F, H, W) + r_lo, plane, n, nr);
        __syncthreads();
        float* dst = out + ((size_t)b * G + grp) * D * plane + (size_t)y * W;
        for (int it = threadIdx.x; it < nx * ndc; it += blockDim.x) {
            const int k = it % nx, d0 = (it / nx) * kDisp, x = x0 + k;
            const int last = min(x, D - 1) - d0;               // disparities d0 + j, j <= last, are computed
            float acc[kDisp];
            {
                const float l = ls[k];
#pragma unroll
                for (int j = 0; j < kDisp; ++j)
                    acc[j] = j <= last ? __fmul_rn(l, rs[x - d0 - j - r_lo]) : 0.f;
            }
            for (int c = 1; c < n; ++c) {
                const float l = ls[c * TX + k];
                const float* rc = rs + c * RP + x - d0 - r_lo;
#pragma unroll
                for (int j = 0; j < kDisp; ++j)
                    if (j <= last) acc[j] = __fadd_rn(acc[j], __fmul_rn(l, rc[-j]));
            }
#pragma unroll
            for (int j = 0; j < kDisp; ++j)
                if (d0 + j < D) dst[(size_t)(d0 + j) * plane + x] = j <= last ? __fdiv_rn(acc[j], fn) : 0.f;
        }
        // planes x0 + nx <= d < D: zero over the tile
        for (int it = threadIdx.x; it < nx * (D - ndc * kDisp); it += blockDim.x) {
            const int k = it % nx, d = ndc * kDisp + it / nx;
            dst[(size_t)d * plane + x0 + k] = 0.f;
        }
    }
}

// ---- gwc backward: grid (x tiles * H, B * G * chunks) ------------------------------------------------------------------
// t = g / n staged twice: tl[d][k] = t[d][x0 + k] for the left gradient and ts[d][k] = t[d][x0 + k + d] for the right one
// (both read along k); then the chunk's right rows [r_lo, x0 + nx) as rs[c][RP] and left rows [x0, x0 + nx + D - 1) as
// ls[c][RP].  A thread owns one (c, x) and both its gradients.
__global__ void __launch_bounds__(kThreads)
gwc_volume_bwd_kernel(const float* __restrict__ L, const float* __restrict__ R, const float* __restrict__ g,
                      float* __restrict__ gl, float* __restrict__ gr, int B, int F, int H, int W, int D, int G, int TX, int RP,
                      int tiles_x) {
    extern __shared__ float4 smem4[];
    const int n = F / G, chunks = (n + kGwcBwdChunk - 1) / kGwcBwdChunk;
    float* tl = reinterpret_cast<float*>(smem4);
    float* ts = tl + (size_t)D * TX;
    float* rs = ts + (size_t)D * TX;
    float* ls = rs + kGwcBwdChunk * RP;
    const int y = (int)(blockIdx.x / tiles_x), x0 = (int)(blockIdx.x % tiles_x) * TX;
    const int nx = min(TX, W - x0), r_lo = max(x0 - D + 1, 0), nr = x0 + nx - r_lo;
    const int nl = min(x0 + nx + D - 1, W) - x0;
    const float fn = (float)n;
    const size_t plane = (size_t)H * W;
    for (long long s = blockIdx.y; s < (long long)B * G * chunks; s += gridDim.y) {
        const int b = (int)(s / ((long long)G * chunks)), grp = (int)(s / chunks % G), chunk = (int)(s % chunks);
        const int c0 = grp * n + chunk * kGwcBwdChunk, nc = min(kGwcBwdChunk, n - chunk * kGwcBwdChunk);
        const float* gt = g + ((size_t)b * G + grp) * D * plane + (size_t)y * W;
        __syncthreads();
        for (int e = threadIdx.x; e < D * nx; e += blockDim.x) {
            const int d = e / nx, k = e % nx, xs = x0 + k + d;
            tl[d * TX + k] = __fdiv_rn(__ldg(gt + (size_t)d * plane + x0 + k), fn);
            ts[d * TX + k] = xs < W ? __fdiv_rn(__ldg(gt + (size_t)d * plane + xs), fn) : 0.f;
        }
        stage_rows(rs, RP, R + row_of(b, c0, y, F, H, W) + r_lo, plane, nc, nr);
        stage_rows(ls, RP, L + row_of(b, c0, y, F, H, W) + x0, plane, nc, nl);
        __syncthreads();
        for (int it = threadIdx.x; it < nc * nx; it += blockDim.x) {
            const int k = it % nx, c = it / nx, x = x0 + k;
            const float* rc = rs + c * RP + x - r_lo;
            const float* lc = ls + c * RP + k;
            const int dl = min(x, D - 1), dr = min(W - 1 - x, D - 1);
            float a = __fmul_rn(tl[k], rc[0]);
            for (int d = 1; d <= dl; ++d) a = __fadd_rn(a, __fmul_rn(tl[d * TX + k], rc[-d]));
            float v = __fmul_rn(ts[k], lc[0]);
            for (int d = 1; d <= dr; ++d) v = __fadd_rn(v, __fmul_rn(ts[d * TX + k], lc[d]));
            const size_t o = row_of(b, c0 + c, y, F, H, W) + x;
            gl[o] = a;
            gr[o] = v;
        }
    }
}

// ---- launch plans --------------------------------------------------------------------------------------------------------
// The tile width TX (a power of two, at most 128 and the first one >= W) and the shared memory of each staged kernel; the
// pitch of a shifted row is RP = min(TX + D - 1, W).  (tests/cost_volume_reference.py restates these plans.)
struct Plan {
    int tx, rp;
    size_t smem;            // 0: no tile fits
};

enum Kind { kConcatFwd, kGwcFwd, kGwcBwd };

size_t smem_of(Kind kind, int tx, int rp, int D, int n) {
    switch (kind) {
        case kConcatFwd: return (size_t)kConcatChunk * (tx + rp) * sizeof(float);
        case kGwcFwd: return (size_t)n * (tx + rp) * sizeof(float);
        default: return ((size_t)2 * D * tx + (size_t)2 * kGwcBwdChunk * rp) * sizeof(float);
    }
}

Plan plan_of(Kind kind, int W, int D, int n) {
    int tx = 1;
    while (tx < 128 && tx < W) tx *= 2;
    for (;; tx /= 2) {
        const int rp = (int)std::min<long long>((long long)tx + D - 1, W);
        const size_t s = smem_of(kind, tx, rp, D, n);
        if (s <= kSmemSoft || (tx == 1 && s <= kSmemHard)) return {tx, rp, s};
        if (tx == 1) return {1, rp, 0};
    }
}

long long ceil_div(long long a, long long b) { return (a + b - 1) / b; }

// Above 48 KB a kernel needs its dynamic shared-memory limit raised.  It is always raised to the same value, the maximum,
// so calls from several host threads cannot lower it under one another's launch (the limit does not change occupancy).
template <class Kernel>
cudaError_t allow_smem(Kernel k, size_t bytes) {
    return bytes > 48 * 1024 ? cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kSmemHard)
                             : cudaSuccess;
}

}  // namespace

int cost_volume_launchable(int F, int H, int W, int D, int G, const char** why) {
    if ((long long)D * H * W >= (1ll << 31)) { *why = "the volume has >= 2^31 elements per (B, channel) slice"; return 0; }
    const bool fits = G == 0 ? plan_of(kConcatFwd, W, D, 0).smem != 0
                             : plan_of(kGwcFwd, W, D, F / G).smem != 0 && plan_of(kGwcBwd, W, D, F / G).smem != 0;
    if (!fits) { *why = "a 1-column tile does not fit in shared memory (D or F / G too large)"; return 0; }
    return 1;
}

int concat_volume_forward(const float* left, const float* right, float* out, int B, int F, int H, int W, int D,
                          cudaStream_t st, int* launches) {
    const Plan p = plan_of(kConcatFwd, W, D, 0);
    const int tiles_x = (int)ceil_div(W, p.tx);
    const int vec = W % 4 == 0 && p.tx % 4 == 0 && (reinterpret_cast<uintptr_t>(out) & 15) == 0;
    CSPN_CUDA_TRY(allow_smem(concat_volume_fwd_kernel, p.smem));
    concat_volume_fwd_kernel<<<dim3((unsigned)((long long)tiles_x * H), slice_blocks((long long)B * ceil_div(F, kConcatChunk))),
                               kThreads, p.smem, st>>>(left, right, out, B, F, H, W, D, p.tx, p.rp, tiles_x, vec);
    CSPN_CUDA_TRY(cudaGetLastError());
    *launches = 1;
    return CSPN_OK;
}

int concat_volume_backward(const float* grad_out, float* grad_left, float* grad_right, int B, int F, int H, int W, int D,
                           cudaStream_t st, int* launches) {
    const long long blocks = std::min<long long>(ceil_div((long long)B * F * H * W, kThreads), 1 << 20);
    concat_volume_bwd_kernel<<<(unsigned)blocks, kThreads, 0, st>>>(grad_out, grad_left, grad_right, B, F, H, W, D);
    CSPN_CUDA_TRY(cudaGetLastError());
    *launches = 1;
    return CSPN_OK;
}

int gwc_volume_forward(const float* left, const float* right, float* out, int B, int F, int H, int W, int D, int G,
                       cudaStream_t st, int* launches) {
    const Plan p = plan_of(kGwcFwd, W, D, F / G);
    const int tiles_x = (int)ceil_div(W, p.tx);
    CSPN_CUDA_TRY(allow_smem(gwc_volume_fwd_kernel, p.smem));
    gwc_volume_fwd_kernel<<<dim3((unsigned)((long long)tiles_x * H), slice_blocks((long long)B * G)), kThreads, p.smem, st>>>(
        left, right, out, B, F, H, W, D, G, p.tx, p.rp, tiles_x);
    CSPN_CUDA_TRY(cudaGetLastError());
    *launches = 1;
    return CSPN_OK;
}

int gwc_volume_backward(const float* left, const float* right, const float* grad_out, float* grad_left, float* grad_right,
                        int B, int F, int H, int W, int D, int G, cudaStream_t st, int* launches) {
    const Plan p = plan_of(kGwcBwd, W, D, F / G);
    const int tiles_x = (int)ceil_div(W, p.tx);
    const long long slices = (long long)B * G * ceil_div(F / G, kGwcBwdChunk);
    CSPN_CUDA_TRY(allow_smem(gwc_volume_bwd_kernel, p.smem));
    gwc_volume_bwd_kernel<<<dim3((unsigned)((long long)tiles_x * H), slice_blocks(slices)), kThreads, p.smem, st>>>(
        left, right, grad_out, grad_left, grad_right, B, F, H, W, D, G, p.tx, p.rp, tiles_x);
    CSPN_CUDA_TRY(cudaGetLastError());
    *launches = 1;
    return CSPN_OK;
}

}  // namespace cspn
