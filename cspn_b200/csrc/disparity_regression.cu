// Disparity regression from a low-resolution cost volume, one op: resize_trilinear to (Do, Ho, Wo), softmax over the
// disparity axis and the expectation sum_o o * p_o, the soft-argmin head of GC-Net / PSMNet-style stereo networks, forward
// and a deterministic backward.  The upsampled volume never reaches memory.
//
//   U = resize_trilinear(cost, (Do, Ho, Wo))       (resize_taps.cuh, the bits of resize_trilinear.cu)
//   y[b,c,h,w] = sum_o o * softmax_o(U[b,c,:,h,w])
//
// Forward, per output pixel, every operation rounded on its own (no FMA contraction):
//   v[d]  = l0h*(l0w*x[d,h0,w0] + l1w*x[d,h0,w1]) + l1h*(l0w*x[d,h1,w0] + l1w*x[d,h1,w1])   for every low-resolution d
//   U_o   = l0d*v[i0(o)] + l1d*v[i1(o)]                                                  (resize's nested order)
//   m     = max_o U_o, NaN if any U_o is NaN
//   S     = sum_o expf(U_o - m),  N = sum_o o * expf(U_o - m)    (ascending o, from 0; expf is the accurate libdevice one)
//   y     = N / S
// A NaN or +inf in the column, or a column all -inf, gives NaN (U - m is NaN somewhere).
// Backward: gU_o = ((expf(U_o - m) * (g / S)) * (o - y)), then resize's adjoint: per pixel along d (gv[d] = sum over the
// outputs o that read d, ascending, of gU_o * w_d), then per low-resolution voxel sum_oh (sum_ow gv[oh,ow][d] * w_w) * w_h,
// each sum from 0 in ascending o, with add_tap's weights (zero-weight taps included, so NaN spreads as in the composition).
//
// Kernels.  The forward is one launch: a CTA owns a TH x TW tile of output pixels of one (b, c) slice, stages the
// low-resolution columns the tile reads (every d) in shared memory, and a thread owns a pixel.  The backward is resize's
// prep launch (the per-axis tap and range tables in the workspace) and one gather launch: a CTA owns a TCH x TCW tile of
// low-resolution cells and every d; it recomputes, for every output pixel that reads one of its cells, the softmax and the
// column adjoint gv[0..D) into shared memory, then one thread per low-resolution voxel sums gv over its window.  Every
// grad_cost element is written once; no atomics, no zero fill, no workspace beyond the tables.
//
// Limits: a tile is shrunk until its shared memory fits; a shape whose 1 x 1 backward tile does not fit in 227 KB is
// CSPN_ERR_UNSUPPORTED, and so is Do > 2^24 (o is counted in fp32).  With Do = D that is D above about 2150 without
// upsampling in H and W (about 4840 when H = W = 1), and above about 520 at 4x in H and W (about 370 with the half-pixel
// rule).  DESIGN.md section 4.15.
#include <cmath>

#include "common.cuh"
#include "resize_taps.cuh"

namespace cspn {
namespace {

constexpr int kThreads = 256;
constexpr size_t kSmemSoft = 110 * 1024;   // two CTAs per SM
constexpr size_t kSmemHard = 227 * 1024;   // the sm_90 per-CTA maximum

// The four staged rows one output pixel blends, as offsets into a plane of the staged block, and its (h, w) weights
struct Column {
    int o00, o01, o10, o11;                // (h0, w0) (h0, w1) (h1, w0) (h1, w1)
    float l0h, l1h, l0w, l1w;
};

__device__ __forceinline__ Column column_of(Tap th, Tap tw, int H, int W, int h_lo, int w_lo, int sw) {
    const int h0 = th.i0 - h_lo, h1 = th.i0 + (th.i0 < H - 1) - h_lo;
    const int w0 = tw.i0 - w_lo, w1 = tw.i0 + (tw.i0 < W - 1) - w_lo;
    return {h0 * sw + w0, h0 * sw + w1, h1 * sw + w0, h1 * sw + w1,
            __fsub_rn(1.f, th.l1), th.l1, __fsub_rn(1.f, tw.l1), tw.l1};
}

// v[d] of resize's nested order: the (h, w) blend of one staged plane
__device__ __forceinline__ float blend_hw(const float* plane, const Column& c) {
    const float a0 = __fadd_rn(__fmul_rn(c.l0w, plane[c.o00]), __fmul_rn(c.l1w, plane[c.o01]));
    const float a1 = __fadd_rn(__fmul_rn(c.l0w, plane[c.o10]), __fmul_rn(c.l1w, plane[c.o11]));
    return __fadd_rn(__fmul_rn(c.l0h, a0), __fmul_rn(c.l1h, a1));
}

// U_o in ascending o.  i0(o) never decreases, so a pass keeps v[i0] and v[i1] and forms each v[d] once (twice where a
// downsampling skips d).
struct Walk {
    const float* xs;
    int plane, D;
    Column c;
    int cur = -2;
    float va = 0.f, vb = 0.f;

    __device__ __forceinline__ float at(Tap t) {
        if (t.i0 != cur) {
            va = t.i0 == cur + 1 ? vb : blend_hw(xs + (size_t)t.i0 * plane, c);
            vb = blend_hw(xs + (size_t)min(t.i0 + 1, D - 1) * plane, c);
            cur = t.i0;
        }
        return __fadd_rn(__fmul_rn(__fsub_rn(1.f, t.l1), va), __fmul_rn(t.l1, vb));
    }
};

struct Soft {
    float m, S, y;
};

// The column's maximum, S and y: two passes over o, shared by the forward and the backward, so both see the same bits
__device__ __forceinline__ Soft regress(const float* xs, int plane, int D, const Column& c, const Tap* dt, int Do) {
    Walk w{xs, plane, D, c};
    float m = -INFINITY;
    for (int o = 0; o < Do; ++o) {
        const float u = w.at(dt[o]);
        m = (u > m || u != u) ? u : m;          // fmaxf would drop a NaN
    }
    Walk w2{xs, plane, D, c};
    float S = 0.f, N = 0.f, fo = 0.f;
    for (int o = 0; o < Do; ++o) {
        const float e = expf(__fsub_rn(w2.at(dt[o]), m));
        S = __fadd_rn(S, e);
        N = __fadd_rn(N, __fmul_rn(fo, e));
        fo = __fadd_rn(fo, 1.f);
    }
    return {m, S, __fdiv_rn(N, S)};
}

// Stages x[bc][0..D)[h_lo, h_lo+sh)[w_lo, w_lo+sw) as xs[d][hh][ww]
__device__ __forceinline__ void stage(float* xs, const float* x, int H, int W, int D, int h_lo, int sh, int w_lo, int sw) {
    const int n = D * sh * sw;
    for (int e = threadIdx.x; e < n; e += blockDim.x) {
        const int ww = e % sw, r = e / sw, hh = r % sh, d = r / sh;
        xs[e] = __ldg(x + ((size_t)d * H + h_lo + hh) * W + w_lo + ww);
    }
}

// ---- forward: grid (output tiles of a slice, slices) -------------------------------------------------------------------
__global__ void __launch_bounds__(kThreads)
disparity_regression_fwd_kernel(const float* __restrict__ x, float* __restrict__ y, long long slices, Axis ad, Axis ah,
                                Axis aw, int TH, int TW, int tiles_w) {
    extern __shared__ float4 smem4[];
    Tap* dt = reinterpret_cast<Tap*>(smem4);
    float* xs = reinterpret_cast<float*>(dt + ad.n_out);
    const int D = ad.n_in, H = ah.n_in, W = aw.n_in, Do = ad.n_out, Ho = ah.n_out, Wo = aw.n_out;
    for (int o = threadIdx.x; o < Do; o += blockDim.x) dt[o] = tap_of(ad, o);
    const int oh0 = (int)(blockIdx.x / tiles_w) * TH, ow0 = (int)(blockIdx.x % tiles_w) * TW;
    const int h_lo = tap_of(ah, oh0).i0, w_lo = tap_of(aw, ow0).i0;
    const Tap th_last = tap_of(ah, min(oh0 + TH, Ho) - 1), tw_last = tap_of(aw, min(ow0 + TW, Wo) - 1);
    const int sh = th_last.i0 + (th_last.i0 < H - 1) - h_lo + 1, sw = tw_last.i0 + (tw_last.i0 < W - 1) - w_lo + 1;
    const int oh = oh0 + (int)threadIdx.x / TW, ow = ow0 + (int)threadIdx.x % TW;
    const bool live = (int)threadIdx.x < TH * TW && oh < Ho && ow < Wo;
    const Column c = column_of(tap_of(ah, min(oh, Ho - 1)), tap_of(aw, min(ow, Wo - 1)), H, W, h_lo, w_lo, sw);
    const size_t vin = (size_t)D * H * W, vout = (size_t)Ho * Wo;
    for (long long bc = blockIdx.y; bc < slices; bc += gridDim.y) {
        __syncthreads();                        // the table is written and the last slice's reads are done
        stage(xs, x + (size_t)bc * vin, H, W, D, h_lo, sh, w_lo, sw);
        __syncthreads();
        if (live) y[(size_t)bc * vout + (size_t)oh * Wo + ow] = regress(xs, sh * sw, D, c, dt, Do).y;
    }
}

// ---- backward, gather: grid (low-resolution cell tiles of a slice, slices) ----------------------------------------------
__global__ void __launch_bounds__(kThreads)
disparity_regression_bwd_kernel(const float* __restrict__ x, const float* __restrict__ g, float* __restrict__ gx,
                                const Tap* __restrict__ taps, const Range* __restrict__ ranges, long long slices, Axis ad,
                                Axis ah, Axis aw, int TCH, int TCW, int tiles_w, int PH, int PW) {
    extern __shared__ float4 smem4[];
    const int D = ad.n_in, H = ah.n_in, W = aw.n_in, Do = ad.n_out, Ho = ah.n_out, Wo = aw.n_out;
    const int Dp = D | 1;                       // an odd column stride: a warp's pixels write different banks
    Tap* dt = reinterpret_cast<Tap*>(smem4);
    Tap* th = dt + Do;
    Tap* tw = th + PH;
    float* xs = reinterpret_cast<float*>(tw + PW);
    float* gv = xs + (size_t)D * (TCH + 2) * (TCW + 2);
    const int ha = (int)(blockIdx.x / tiles_w) * TCH, wa = (int)(blockIdx.x % tiles_w) * TCW;
    const int nch = min(TCH, H - ha), ncw = min(TCW, W - wa);
    const Range* rh = ranges + D;
    const Range* rw = ranges + D + H;
    // the output pixels that read a cell of the tile: [oh_b, oh_b + ph) x [ow_b, ow_b + pw), ph <= PH and pw <= PW
    const int oh_b = rh[ha].b, ph = rh[ha + nch - 1].e - oh_b, ow_b = rw[wa].b, pw = rw[wa + ncw - 1].e - ow_b;
    // they read the rows [ha - 1, ha + nch] and columns [wa - 1, wa + ncw], clipped
    const int h_lo = max(ha - 1, 0), sh = min(ha + nch, H - 1) - h_lo + 1;
    const int w_lo = max(wa - 1, 0), sw = min(wa + ncw, W - 1) - w_lo + 1;
    for (int o = threadIdx.x; o < Do; o += blockDim.x) dt[o] = taps[o];
    for (int k = threadIdx.x; k < ph; k += blockDim.x) th[k] = taps[Do + oh_b + k];
    for (int k = threadIdx.x; k < pw; k += blockDim.x) tw[k] = taps[Do + Ho + ow_b + k];
    const size_t vin = (size_t)D * H * W, vout = (size_t)Ho * Wo;
    for (long long bc = blockIdx.y; bc < slices; bc += gridDim.y) {
        __syncthreads();
        stage(xs, x + (size_t)bc * vin, H, W, D, h_lo, sh, w_lo, sw);
        __syncthreads();
        // phase 1: a thread per output pixel recomputes the softmax and writes the column adjoint gv[0..D)
        for (int p = threadIdx.x; p < ph * pw; p += blockDim.x) {
            const int kh = p / pw, kw = p % pw;
            const Column c = column_of(th[kh], tw[kw], H, W, h_lo, w_lo, sw);
            const Soft s = regress(xs, sh * sw, D, c, dt, Do);
            const float q = __fdiv_rn(__ldg(g + (size_t)bc * vout + (size_t)(oh_b + kh) * Wo + ow_b + kw), s.S);
            float* col = gv + (size_t)p * Dp;
            for (int d = 0; d < D; ++d) col[d] = 0.f;          // indices no output reads (a downsampling in d)
            Walk w{xs, sh * sw, D, c};
            int cur = dt[0].i0;
            float ga = 0.f, gb = 0.f;                            // the sums of indices cur and cur + 1
            float fo = 0.f;
            for (int o = 0; o < Do; ++o) {
                const Tap t = dt[o];
                const float gu = __fmul_rn(__fmul_rn(expf(__fsub_rn(w.at(t), s.m)), q), __fsub_rn(fo, s.y));
                fo = __fadd_rn(fo, 1.f);
                if (t.i0 != cur) {                               // index cur has all its outputs
                    col[cur] = ga;
                    if (t.i0 == cur + 1) {
                        ga = gb;
                    } else {
                        if (cur + 1 < D) col[cur + 1] = gb;
                        ga = 0.f;
                    }
                    gb = 0.f;
                    cur = t.i0;
                }
                ga = __fadd_rn(ga, __fmul_rn(gu, __fsub_rn(1.f, t.l1)));
                if (cur == D - 1) ga = __fadd_rn(ga, __fmul_rn(gu, t.l1));
                else gb = __fadd_rn(gb, __fmul_rn(gu, t.l1));
            }
            col[cur] = ga;
            if (cur + 1 < D) col[cur + 1] = gb;
        }
        __syncthreads();
        // phase 2: a thread per low-resolution voxel, d fastest: sum_oh (sum_ow gv * w_w) * w_h, ascending
        for (int v = threadIdx.x; v < D * nch * ncw; v += blockDim.x) {
            const int d = v % D, cell = v / D, h = ha + cell / ncw, w = wa + cell % ncw;
            const Range ry = rh[h], rx = rw[w];
            float acc_h = 0.f;
            for (int oh = ry.b; oh < ry.e; ++oh) {
                const float* row = gv + (size_t)(oh - oh_b) * pw * Dp + d;
                float acc_w = 0.f;
                for (int ow = rx.b; ow < rx.e; ++ow)
                    acc_w = add_tap(acc_w, row[(size_t)(ow - ow_b) * Dp], tw[ow - ow_b], w, W);
                acc_h = add_tap(acc_h, acc_w, th[oh - oh_b], h, H);
            }
            gx[(size_t)bc * vin + ((size_t)d * H + h) * W + w] = acc_h;
        }
    }
}

// ---- launch plans --------------------------------------------------------------------------------------------------------
// An upper bound of the low-resolution indices that t consecutive outputs read along an axis: the source coordinates of
// the first and last differ by r*(t-1) up to fp32 rounding, plus i1 and the floor of each end
int span_in(const Axis& a, int t) {
    const double s = (double)a.r * (t - 1) + (a.n_in + 2.0) * std::ldexp(1.0, -21);
    return (int)std::min<double>(a.n_in, std::floor(s) + 3);
}

// An upper bound of the outputs that read t consecutive low-resolution indices i..i+t-1 along an axis: those with
// i0 in [i-1, i+t-1], whose source coordinates lie in [i-1, i+t+1), an interval of length t+1.  With the half-pixel rule
// the coordinate r*(o+0.5)-0.5 is clamped at 0, so for i <= 1 the outputs with a coordinate in [-0.5, 0) read index 0 too:
// the interval is [-0.5, i+t+1), at most t+1.5 long.  An interval of length L holds at most L/r outputs and one more;
// fp32 rounding moves each coordinate by at most 4u*n_out outputs' worth, and one more output covers the ends.
// (tests/disparity_reference.py restates span_in, span_out and the plans, and checks them against the fp32 taps.)
int span_out(const Axis& a, int t) {
    if (a.r == 0.f) return a.n_out;
    const double len = t + 1.0 + (a.half ? 0.5 : 0.0);
    const double s = len / (double)a.r + (a.n_out + 2.0) * std::ldexp(1.0, -21);
    return (int)std::min<double>(a.n_out, std::floor(s) + 2);
}

struct Plan {
    int th, tw;             // the tile: output pixels (forward) or low-resolution cells (backward)
    int ph, pw;             // backward: the bounds of the output pixels that read the tile
    size_t smem;
};

size_t fwd_smem(const Axis& ad, const Axis& ah, const Axis& aw, int th, int tw) {
    return (size_t)ad.n_out * sizeof(Tap) + (size_t)ad.n_in * span_in(ah, th) * span_in(aw, tw) * sizeof(float);
}

Plan bwd_plan_for(const Axis& ad, const Axis& ah, const Axis& aw, int th, int tw) {
    const int ph = span_out(ah, th), pw = span_out(aw, tw);
    const size_t smem = ((size_t)ad.n_out + ph + pw) * sizeof(Tap) + (size_t)ad.n_in * (th + 2) * (tw + 2) * sizeof(float) +
                        (size_t)ph * pw * (ad.n_in | 1) * sizeof(float);
    return {th, tw, ph, pw, smem};
}

// The first tile that fits two CTAs per SM, else the smallest if it fits at all; smem == 0 when none fits
Plan fwd_plan(const Axis& ad, const Axis& ah, const Axis& aw) {
    static const int tiles[][2] = {{8, 32}, {4, 32}, {2, 32}, {1, 32}, {1, 16}, {1, 8}, {1, 4}, {1, 2}, {1, 1}};
    for (const auto& t : tiles) {
        const size_t s = fwd_smem(ad, ah, aw, t[0], t[1]);
        if (s <= kSmemSoft || (t[0] == 1 && t[1] == 1 && s <= kSmemHard)) return {t[0], t[1], 0, 0, s};
    }
    return {1, 1, 0, 0, 0};
}

Plan bwd_plan(const Axis& ad, const Axis& ah, const Axis& aw) {
    static const int tiles[][2] = {{8, 8}, {4, 8}, {4, 4}, {2, 4}, {2, 2}, {1, 2}, {1, 1}};
    for (const auto& t : tiles) {
        const Plan p = bwd_plan_for(ad, ah, aw, t[0], t[1]);
        if (p.smem <= kSmemSoft || (t[0] == 1 && t[1] == 1 && p.smem <= kSmemHard)) return p;
    }
    return {1, 1, 0, 0, 0};
}

int ceil_div(int a, int b) { return (a + b - 1) / b; }

// Above 48 KB a kernel needs its dynamic shared-memory limit raised.  It is always raised to the same value, the maximum,
// so calls from several host threads cannot lower it under one another's launch (the limit does not change occupancy).
template <class Kernel>
cudaError_t allow_smem(Kernel k, size_t bytes) {
    return bytes > 48 * 1024 ? cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kSmemHard)
                             : cudaSuccess;
}

}  // namespace

int disparity_regression_launchable(int D, int H, int W, int Do, int Ho, int Wo, int align_corners, int align_mode,
                                    const char** why) {
    if (Do > (1 << 24)) { *why = "Do > 2^24 (disparities are counted in fp32)"; return 0; }
    const Axis ad = make_axis(D, Do, align_corners, align_mode), ah = make_axis(H, Ho, align_corners, align_mode);
    const Axis aw = make_axis(W, Wo, align_corners, align_mode);
    if (!fwd_plan(ad, ah, aw).smem || !bwd_plan(ad, ah, aw).smem) {
        *why = "a 1x1 tile of the cost columns does not fit in shared memory (D or Do too large)";
        return 0;
    }
    return 1;
}

int disparity_regression_forward(const float* cost, float* out, long long slices, int D, int H, int W, int Do, int Ho, int Wo,
                                 int align_corners, int align_mode, cudaStream_t st, int* launches) {
    const Axis ad = make_axis(D, Do, align_corners, align_mode), ah = make_axis(H, Ho, align_corners, align_mode);
    const Axis aw = make_axis(W, Wo, align_corners, align_mode);
    const Plan p = fwd_plan(ad, ah, aw);
    const int tiles_w = ceil_div(Wo, p.tw);
    CSPN_CUDA_TRY(allow_smem(disparity_regression_fwd_kernel, p.smem));
    disparity_regression_fwd_kernel<<<dim3((unsigned)(ceil_div(Ho, p.th) * (long long)tiles_w), slice_blocks(slices)), kThreads,
                                      p.smem, st>>>(cost, out, slices, ad, ah, aw, p.th, p.tw, tiles_w);
    CSPN_CUDA_TRY(cudaGetLastError());
    *launches = 1;
    return CSPN_OK;
}

int disparity_regression_backward(const float* cost, const float* grad_out, float* grad_cost, long long slices, int D, int H,
                                  int W, int Do, int Ho, int Wo, int align_corners, int align_mode, void* ws, cudaStream_t st,
                                  int* launches) {
    const Axis ad = make_axis(D, Do, align_corners, align_mode), ah = make_axis(H, Ho, align_corners, align_mode);
    const Axis aw = make_axis(W, Wo, align_corners, align_mode);
    const Plan p = bwd_plan(ad, ah, aw);
    const Range* ranges = launch_resize_prep(ws, ad, ah, aw, st);
    CSPN_CUDA_TRY(cudaGetLastError());
    const int tiles_w = ceil_div(W, p.tw);
    CSPN_CUDA_TRY(allow_smem(disparity_regression_bwd_kernel, p.smem));
    disparity_regression_bwd_kernel<<<dim3((unsigned)(ceil_div(H, p.th) * (long long)tiles_w), slice_blocks(slices)), kThreads,
                                      p.smem, st>>>(cost, grad_out, grad_cost, static_cast<const Tap*>(ws), ranges, slices,
                                                    ad, ah, aw, p.th, p.tw, tiles_w, p.ph, p.pw);
    CSPN_CUDA_TRY(cudaGetLastError());
    *launches = 2;
    return CSPN_OK;
}

}  // namespace cspn
