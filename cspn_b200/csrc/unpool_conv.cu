// The guidance and depth heads of the reference model (Simple_Gudi_UpConv_Block_Last_Layer,
// /root/reference/cspn_pytorch/models/torch_resnet_cspn_nyu.py:187-205): Unpool (a [1,0;0,0] conv_transpose2d, stride 2,
// :41-54), a crop to (H, W), and a 3x3 convolution with zero padding -- in one polyphase kernel, and its backward.
//
// Polyphase form.  With u the zero-inserted map cropped to H x W (u(2i, 2j) = x(i, j), every other cell x(i, j) * 0),
// output row 2i reads source row i only (tap row 1) and output row 2i+1 reads rows i (tap row 0) and i+1 (tap row 2, only
// if 2i+2 < H); the same holds for columns.  So the 2x2 output block anchored at source (i, j) needs the source window
// (i..i+1, j..j+1) and 9 products per input channel, against 36 over the zero-inserted map:
//   out(2i,   2j)   = sum_ci w11 x(i,j)
//   out(2i,   2j+1) = sum_ci w10 x(i,j) + w12 x(i,j+1)
//   out(2i+1, 2j)   = sum_ci w01 x(i,j) + w21 x(i+1,j)
//   out(2i+1, 2j+1) = sum_ci w00 x(i,j) + w02 x(i,j+1) + w20 x(i+1,j) + w22 x(i+1,j+1)
// Source cells with 2i >= H or 2j >= W are cropped away: they are staged as 0, which is what the padding gives.
//
// IEEE.  The products skipped above are w * (x * 0) (inserted cells) and w * 0 (padding).  They are zero for finite
// operands; otherwise they are NaN, and so is the output that sums them.  The forward puts those NaNs back: a per-CTA flag
// "some x of the staged window is non-finite" and a per-output-channel 9-bit mask "tap t is non-finite for some input
// channel" select a cold path that rebuilds each output's set of structural-zero taps.  Finite inputs never take it.
//
// Backward.  grad_x(ci, i, j) = sum_co sum_tap w[co, ci, tap] g(co, 2i+1-ky, 2j+1-kx) over in-range outputs, a gather (no
// atomics), 0 where the crop removes (i, j).  grad_w[co, ci, tap] = sum over the surviving source pixels of
// x(ci, i, j) g(co, 2i+1-ky, 2j+1-kx): per-CTA partials over fixed pixel ranges go to the workspace, then a second kernel
// sums them in CTA order.  Only the real cells carry gradient: a non-finite grad_out is not multiplied by the structural
// zeros the op sequence's autograd would multiply it by, so non-finite values do not spread to where autograd would put NaN.
// Every sum has a fixed order, so the forward and grad_x bits of an image do not depend on the rest of the batch, and
// grad_w is the same from run to run.
#include "common.cuh"

namespace cspn {
namespace {

constexpr int kThreads = 256;            // 32 x 8: a thread owns source column tx, rows 2ty and 2ty+1 of its tile
constexpr int kTH = 16, kTW = 32;        // source tile of the forward and grad_x kernels
constexpr int kSR = kTH + 2, kSC = kTW + 2;   // staged rows / cols: one halo row / col on each side
constexpr int kCiChunk = 16;             // input channels staged at a time (forward)
constexpr int kCoChunk = 16;             // output channels of weights staged at a time (grad_x)
constexpr int kCig = 8;                  // input channels per CTA (grad_x)
constexpr int kKP = 32;                  // source pixels per staged chunk (grad_w)
constexpr int kWgradCtas = 528;          // grad_w partial CTAs aimed at: 4 per SM of an H100 SXM

// tap t = 3*ky + kx of the 2x2 block: which output (0: (2i,2j), 1: (2i,2j+1), 2: (2i+1,2j), 3: (2i+1,2j+1)) it feeds and
// which source value it reads (0: (i,j), 1: (i,j+1), 2: (i+1,j), 3: (i+1,j+1))
__host__ __device__ constexpr int tap_out(int t) { return t == 4 ? 0 : (t == 3 || t == 5) ? 1 : (t == 1 || t == 7) ? 2 : 3; }
__host__ __device__ constexpr int tap_src(int t) { return t == 2 || t == 5 ? 1 : (t == 6 || t == 7) ? 2 : t == 8 ? 3 : 0; }

__device__ __forceinline__ float qnan() { return __int_as_float(0x7fffffff); }

template <int N>
__device__ __forceinline__ void load_vec(float (&v)[N], const float* p) {
    if constexpr (N % 4 == 0) {
#pragma unroll
        for (int k = 0; k < N; k += 4) {
            const float4 q = *reinterpret_cast<const float4*>(p + k);
            v[k] = q.x, v[k + 1] = q.y, v[k + 2] = q.z, v[k + 3] = q.w;
        }
    } else {
#pragma unroll
        for (int k = 0; k < N; ++k) v[k] = p[k];
    }
}

// ---- forward: grid (source tiles, groups of COG output channels, images) ----------------------------------------------
template <int COG>
__global__ void __launch_bounds__(kThreads, 2)
unpool_conv_fwd_kernel(const float* __restrict__ x, const float* __restrict__ w, float* __restrict__ out, int Cin, int h,
                       int wd, int Cout, int H, int W, int tiles_x) {
    __shared__ float xs[kCiChunk][kSR][kSC];
    __shared__ __align__(16) float wsm[kCiChunk][9][COG];
    __shared__ unsigned char bad[kSR][kSC];          // the source cell is non-finite in some input channel
    __shared__ unsigned wmask[COG];                  // bit t: tap t is non-finite for some input channel
    const int tid = threadIdx.x, tx = tid & 31, ty = tid >> 5;
    const int co0 = blockIdx.y * COG, b = blockIdx.z, nco = min(COG, Cout - co0);
    const int i0 = (blockIdx.x / tiles_x) * kTH, j0 = (blockIdx.x % tiles_x) * kTW;
    const int hv = (H + 1) >> 1, wv = (W + 1) >> 1;  // source rows / cols that survive the crop
    for (int e = tid; e < kSR * kSC; e += kThreads) (&bad[0][0])[e] = 0;
    if (tid < COG) wmask[tid] = 0u;
    float acc[2][4][COG];
#pragma unroll
    for (int p = 0; p < 2; ++p)
#pragma unroll
        for (int q = 0; q < 4; ++q)
#pragma unroll
            for (int c = 0; c < COG; ++c) acc[p][q][c] = 0.f;
    const float* xb = x + (size_t)b * Cin * h * wd;
    int saw_bad = 0;
    const int r = 1 + 2 * ty, c = 1 + tx;            // staged position of the thread's first source pixel
    for (int c0 = 0; c0 < Cin; c0 += kCiChunk) {
        const int nc = min(kCiChunk, Cin - c0);
        __syncthreads();                             // the previous chunk is consumed (and bad / wmask are cleared)
        for (int e = tid; e < kCiChunk * kSR * kSC; e += kThreads) {
            const int cl = e / (kSR * kSC), rc = e - cl * (kSR * kSC), sr = rc / kSC, sc = rc - sr * kSC;
            const int i = i0 - 1 + sr, j = j0 - 1 + sc;
            float v = 0.f;
            if (cl < nc && i >= 0 && j >= 0 && i < hv && j < wv) {
                v = __ldg(xb + ((size_t)(c0 + cl) * h + i) * wd + j);
                if (!isfinite(v)) bad[sr][sc] = 1, saw_bad = 1;
            }
            xs[cl][sr][sc] = v;
        }
        for (int e = tid; e < COG * kCiChunk * 9; e += kThreads) {
            const int co = e / (kCiChunk * 9), rem = e - co * (kCiChunk * 9), cl = rem / 9, t = rem - cl * 9;
            float v = 0.f;
            if (cl < nc && co < nco) {
                v = __ldg(w + ((size_t)(co0 + co) * Cin + c0 + cl) * 9 + t);
                if (!isfinite(v)) atomicOr(&wmask[co], 1u << t);
            }
            wsm[cl][t][co] = v;
        }
        __syncthreads();
        for (int cl = 0; cl < nc; ++cl) {
            float s[2][4];
#pragma unroll
            for (int p = 0; p < 2; ++p) {
                s[p][0] = xs[cl][r + p][c];
                s[p][1] = xs[cl][r + p][c + 1];
                s[p][2] = xs[cl][r + p + 1][c];
                s[p][3] = xs[cl][r + p + 1][c + 1];
            }
#pragma unroll
            for (int t = 0; t < 9; ++t) {
                float wv_[COG];
                load_vec(wv_, &wsm[cl][t][0]);
#pragma unroll
                for (int p = 0; p < 2; ++p)
#pragma unroll
                    for (int k = 0; k < COG; ++k) acc[p][tap_out(t)][k] = fmaf(wv_[k], s[p][tap_src(t)], acc[p][tap_out(t)][k]);
            }
        }
    }
    unsigned wany = 0u;
#pragma unroll
    for (int k = 0; k < COG; ++k) wany |= wmask[k];
    const bool cold = __syncthreads_or(saw_bad) || wany;
    float* ob = out + ((size_t)b * Cout + co0) * H * W;
#pragma unroll
    for (int p = 0; p < 2; ++p) {
        const int i = i0 + 2 * ty + p, j = j0 + tx;
        if (i >= hv || j >= wv) continue;
#pragma unroll
        for (int q = 0; q < 4; ++q) {
            const int oy = 2 * i + (q >> 1), ox = 2 * j + (q & 1);
            if (oy >= H || ox >= W) continue;
            if (cold) {                              // rebuild the NaNs of the products skipped as structural zeros
                unsigned zero_taps = 0u;
                bool xnan = false;
                for (int t = 0; t < 9; ++t) {
                    const int uy = oy + t / 3 - 1, ux = ox + t % 3 - 1;
                    if (uy < 0 || ux < 0 || uy >= H || ux >= W) {
                        zero_taps |= 1u << t;                        // padding: w * 0
                    } else if ((uy | ux) & 1) {
                        zero_taps |= 1u << t;                        // inserted cell: w * (x * 0)
                        xnan |= bad[(uy >> 1) - i0 + 1][(ux >> 1) - j0 + 1] != 0;
                    }
                }
#pragma unroll
                for (int k = 0; k < COG; ++k)
                    if (xnan || (wmask[k] & zero_taps)) acc[p][q][k] = qnan();
            }
#pragma unroll
            for (int k = 0; k < COG; ++k)
                if (k < nco) ob[((size_t)k * H + oy) * W + ox] = acc[p][q][k];
        }
    }
}

// ---- grad_x: grid (source tiles over the whole h x w, groups of kCig input channels, images) ---------------------------
__global__ void __launch_bounds__(kThreads, 2)
unpool_conv_dgrad_kernel(const float* __restrict__ g, const float* __restrict__ w, float* __restrict__ gx, int Cin, int h,
                         int wd, int Cout, int H, int W, int tiles_x) {
    __shared__ __align__(16) float wsm[kCoChunk][9][kCig];
    const int tid = threadIdx.x, tx = tid & 31, ty = tid >> 5;
    const int ci0 = blockIdx.y * kCig, b = blockIdx.z, nci = min(kCig, Cin - ci0);
    const int i = (blockIdx.x / tiles_x) * kTH + 2 * ty, j = (blockIdx.x % tiles_x) * kTW + tx;
    const int hv = (H + 1) >> 1, wv = (W + 1) >> 1;
    float acc[2][kCig];
#pragma unroll
    for (int p = 0; p < 2; ++p)
#pragma unroll
        for (int k = 0; k < kCig; ++k) acc[p][k] = 0.f;
    // the thread's grad_out window: rows 2i-1 .. 2i+3, cols 2j-1 .. 2j+1 (row 2p+2-ky, col 2-kx for pixel p and tap)
    int roff[5], coff[3];
    bool rok[5], cok[3];
#pragma unroll
    for (int k = 0; k < 5; ++k) {
        const int y = 2 * i - 1 + k;
        rok[k] = y >= 0 && y < H;
        roff[k] = y * W;
    }
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        const int xx = 2 * j - 1 + k;
        cok[k] = xx >= 0 && xx < W && j < wv;
        coff[k] = xx;
    }
    const bool live = i < hv && j < wv;
    const float* gb = g + (size_t)b * Cout * H * W;
    for (int c0 = 0; c0 < Cout; c0 += kCoChunk) {
        const int nco = min(kCoChunk, Cout - c0);
        __syncthreads();
        for (int e = tid; e < kCoChunk * kCig * 9; e += kThreads) {
            const int col = e / (kCig * 9), rem = e - col * (kCig * 9), cil = rem / 9, t = rem - cil * 9;
            float v = 0.f;
            if (col < nco && cil < nci) v = __ldg(w + ((size_t)(c0 + col) * Cin + ci0 + cil) * 9 + t);
            wsm[col][t][cil] = v;
        }
        __syncthreads();
        if (!live) continue;
        for (int col = 0; col < nco; ++col) {
            const float* gc = gb + (size_t)(c0 + col) * H * W;
            float gw[5][3];
#pragma unroll
            for (int a = 0; a < 5; ++a)
#pragma unroll
                for (int k = 0; k < 3; ++k) gw[a][k] = (rok[a] && cok[k]) ? __ldg(gc + roff[a] + coff[k]) : 0.f;
#pragma unroll
            for (int t = 0; t < 9; ++t) {
                float wv_[kCig];
                load_vec(wv_, &wsm[col][t][0]);
#pragma unroll
                for (int p = 0; p < 2; ++p) {
                    const float gv = gw[2 * p + 2 - t / 3][2 - t % 3];
#pragma unroll
                    for (int k = 0; k < kCig; ++k) acc[p][k] = fmaf(wv_[k], gv, acc[p][k]);
                }
            }
        }
    }
#pragma unroll
    for (int p = 0; p < 2; ++p) {
        const int ii = i + p;
        if (ii >= h || j >= wd) continue;
        const bool in_crop = ii < hv && j < wv;
#pragma unroll
        for (int k = 0; k < kCig; ++k)
            if (k < nci) gx[(((size_t)b * Cin + ci0 + k) * h + ii) * wd + j] = in_crop ? acc[p][k] : 0.f;
    }
}

// ---- grad_w, pass 1: grid (pixel ranges, groups of COG output channels, groups of 32 input channels) --------------------
// The surviving source pixels (b, i < hv, j < wv) are numbered b-major; CTA n sums pixels [n*per_cta, (n+1)*per_cta) in
// chunks of kKP.  Warp wp owns output channel wp % COG and every (8/COG)-th pixel of a chunk from wp / COG on, lane l
// input channel l: 9 accumulators, one per tap.  The 8/COG slices are added in slice order at the end.
template <int COG>
__global__ void __launch_bounds__(kThreads)
unpool_conv_wgrad_partial_kernel(const float* __restrict__ x, const float* __restrict__ g, float* __restrict__ part, int Cin,
                                 int h, int wd, int Cout, int H, int W, long long npix, long long per_cta) {
    constexpr int KS = 8 / COG;
    __shared__ float xs[kKP][32];
    __shared__ float gs[kKP][COG][9];
    __shared__ float red[8][9][32];
    const int tid = threadIdx.x, lane = tid & 31, wp = tid >> 5, col = wp % COG, ks = wp / COG;
    const int co0 = blockIdx.y * COG, ci0 = blockIdx.z * 32;
    const int hv = (H + 1) >> 1, wv = (W + 1) >> 1;
    const long long pb = (long long)blockIdx.x * per_cta, pe = min(npix, pb + per_cta);
    float acc[9];
#pragma unroll
    for (int t = 0; t < 9; ++t) acc[t] = 0.f;
    for (long long p0 = pb; p0 < pe; p0 += kKP) {
        __syncthreads();
        for (int e = tid; e < kKP * 32; e += kThreads) {
            const int k = e % kKP, cl = e / kKP;
            const long long pp = p0 + k;
            float v = 0.f;
            if (pp < pe && ci0 + cl < Cin) {
                const int j = (int)(pp % wv);
                const long long rest = pp / wv;
                const int i = (int)(rest % hv), b = (int)(rest / hv);
                v = __ldg(x + (((size_t)b * Cin + ci0 + cl) * h + i) * wd + j);
            }
            xs[k][cl] = v;
        }
        for (int e = tid; e < kKP * COG * 9; e += kThreads) {
            const int k = e % kKP, rem = e / kKP, t = rem % 9, cl = rem / 9;
            const long long pp = p0 + k;
            float v = 0.f;
            if (pp < pe && co0 + cl < Cout) {
                const int j = (int)(pp % wv);
                const long long rest = pp / wv;
                const int i = (int)(rest % hv), b = (int)(rest / hv);
                const int oy = 2 * i + 1 - t / 3, ox = 2 * j + 1 - t % 3;
                if (oy >= 0 && ox >= 0 && oy < H && ox < W) v = __ldg(g + (((size_t)b * Cout + co0 + cl) * H + oy) * W + ox);
            }
            gs[k][cl][t] = v;
        }
        __syncthreads();
        for (int k = ks; k < kKP; k += KS) {
            const float xv = xs[k][lane];
#pragma unroll
            for (int t = 0; t < 9; ++t) acc[t] = fmaf(gs[k][col][t], xv, acc[t]);
        }
    }
    if constexpr (KS > 1) {
#pragma unroll
        for (int t = 0; t < 9; ++t) red[wp][t][lane] = acc[t];
        __syncthreads();
        if (ks == 0)
            for (int s = 1; s < KS; ++s)
#pragma unroll
                for (int t = 0; t < 9; ++t) acc[t] += red[col + s * COG][t][lane];
    }
    if (ks == 0 && co0 + col < Cout && ci0 + lane < Cin) {
        float* dst = part + (((size_t)blockIdx.x * Cout + co0 + col) * Cin + ci0 + lane) * 9;
#pragma unroll
        for (int t = 0; t < 9; ++t) dst[t] = acc[t];
    }
}

// ---- grad_w, pass 2: the partials summed in CTA order -------------------------------------------------------------------
__global__ void __launch_bounds__(kThreads)
unpool_conv_wgrad_reduce_kernel(const float* __restrict__ part, float* __restrict__ gw, size_t n, int nparts) {
    for (size_t e = (size_t)blockIdx.x * kThreads + threadIdx.x; e < n; e += (size_t)gridDim.x * kThreads) {
        float s = part[e];
        for (int q = 1; q < nparts; ++q) s += part[(size_t)q * n + e];
        gw[e] = s;
    }
}

int pick_group(int C) { return C >= 5 ? 8 : C >= 3 ? 4 : C; }

template <int COG>
void launch_fwd(const float* x, const float* w, float* out, int B, int Cin, int h, int wd, int Cout, int H, int W,
                cudaStream_t st) {
    const int hv = (H + 1) / 2, wv = (W + 1) / 2, tx = (wv + kTW - 1) / kTW, ty = (hv + kTH - 1) / kTH;
    unpool_conv_fwd_kernel<COG><<<dim3(tx * ty, (Cout + COG - 1) / COG, B), kThreads, 0, st>>>(x, w, out, Cin, h, wd, Cout, H, W, tx);
}

template <int COG>
void launch_wgrad(const float* x, const float* g, float* part, int Cin, int h, int wd, int Cout, int H, int W, long long npix,
                  long long per_cta, int nparts, cudaStream_t st) {
    unpool_conv_wgrad_partial_kernel<COG><<<dim3(nparts, (Cout + COG - 1) / COG, (Cin + 31) / 32), kThreads, 0, st>>>(
        x, g, part, Cin, h, wd, Cout, H, W, npix, per_cta);
}

}  // namespace

// The pixel split of grad_w: per_cta pixels (a multiple of kKP) for each of *nparts CTAs.  Depends on the shape only.
void unpool_conv_wgrad_plan(int B, int Cin, int H, int W, int Cout, long long* per_cta, int* nparts) {
    const long long npix = (long long)B * ((H + 1) / 2) * ((W + 1) / 2);
    const long long chunks = (npix + kKP - 1) / kKP;
    const long long groups = (long long)((Cout + pick_group(Cout) - 1) / pick_group(Cout)) * ((Cin + 31) / 32);
    long long want = (kWgradCtas + groups - 1) / groups;
    if (want < 1) want = 1;
    if (want > chunks) want = chunks;
    const long long cpc = (chunks + want - 1) / want;
    *per_cta = cpc * kKP;
    *nparts = (int)((chunks + cpc - 1) / cpc);
}

size_t unpool_conv_bwd_workspace_bytes(int B, int Cin, int H, int W, int Cout) {
    long long per_cta;
    int nparts;
    unpool_conv_wgrad_plan(B, Cin, H, W, Cout, &per_cta, &nparts);
    return (size_t)nparts * Cout * Cin * 9 * sizeof(float);
}

int unpool_conv_launchable(int B, int Cin, int Cout, const char** why) {
    if (B > 65535) { *why = "B > 65535 (gridDim.z)"; return 0; }
    if ((Cout + pick_group(Cout) - 1) / pick_group(Cout) > 65535 || (Cin + kCig - 1) / kCig > 65535) { *why = "too many channels for gridDim.y"; return 0; }
    return 1;
}

int unpool_conv_forward(const float* x, const float* w, float* out, int B, int Cin, int h, int wd, int Cout, int H, int W,
                        cudaStream_t st, int* launches) {
    switch (pick_group(Cout)) {
        case 1: launch_fwd<1>(x, w, out, B, Cin, h, wd, Cout, H, W, st); break;
        case 2: launch_fwd<2>(x, w, out, B, Cin, h, wd, Cout, H, W, st); break;
        case 4: launch_fwd<4>(x, w, out, B, Cin, h, wd, Cout, H, W, st); break;
        default: launch_fwd<8>(x, w, out, B, Cin, h, wd, Cout, H, W, st); break;
    }
    CSPN_CUDA_TRY(cudaGetLastError());
    *launches = 1;
    return CSPN_OK;
}

int unpool_conv_backward(const float* x, const float* w, const float* g, float* gx, float* gw, int B, int Cin, int h, int wd,
                         int Cout, int H, int W, void* ws, cudaStream_t st, int* launches) {
    int n = 0;
    if (gx) {
        const int tx = (wd + kTW - 1) / kTW, ty = (h + kTH - 1) / kTH;
        unpool_conv_dgrad_kernel<<<dim3(tx * ty, (Cin + kCig - 1) / kCig, B), kThreads, 0, st>>>(g, w, gx, Cin, h, wd, Cout, H, W, tx);
        CSPN_CUDA_TRY(cudaGetLastError());
        ++n;
    }
    if (gw) {
        long long per_cta;
        int nparts;
        unpool_conv_wgrad_plan(B, Cin, H, W, Cout, &per_cta, &nparts);
        const long long npix = (long long)B * ((H + 1) / 2) * ((W + 1) / 2);
        float* part = static_cast<float*>(ws);
        switch (pick_group(Cout)) {
            case 1: launch_wgrad<1>(x, g, part, Cin, h, wd, Cout, H, W, npix, per_cta, nparts, st); break;
            case 2: launch_wgrad<2>(x, g, part, Cin, h, wd, Cout, H, W, npix, per_cta, nparts, st); break;
            case 4: launch_wgrad<4>(x, g, part, Cin, h, wd, Cout, H, W, npix, per_cta, nparts, st); break;
            default: launch_wgrad<8>(x, g, part, Cin, h, wd, Cout, H, W, npix, per_cta, nparts, st); break;
        }
        CSPN_CUDA_TRY(cudaGetLastError());
        const size_t ne = (size_t)Cout * Cin * 9;
        const size_t blocks = (ne + kThreads - 1) / kThreads;
        unpool_conv_wgrad_reduce_kernel<<<(unsigned)(blocks < 1024 ? blocks : 1024), kThreads, 0, st>>>(part, gw, ne, nparts);
        CSPN_CUDA_TRY(cudaGetLastError());
        n += 2;
    }
    *launches = n;
    return CSPN_OK;
}

}  // namespace cspn
