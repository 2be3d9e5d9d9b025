// Trilinear resampling of volumes, the Paddle module's `resize_trilinear` (fluid.layers.resize_trilinear, one of the two
// custom ops of the Paddle wheel the reference's Paddle half is built on), forward and a deterministic backward.
//
// Per axis, n_in -> n_out, in fp32 with every operation rounded on its own (__fmul_rn / __fadd_rn / __fsub_rn: no FMA
// contraction, so tests/resize_reference.py restates the bits in numpy):
//   r = (n_in-1)/(n_out-1) with align_corners, else n_in/n_out; r = 0 when n_out == 1 (computed once on the host)
//   s(o) = max(r*(o+0.5) - 0.5, 0) with align_corners off and align_mode 0, else r*o
//   i0 = (int)s, i1 = i0 + (i0 < n_in-1), l1 = s - i0, l0 = 1 - l1
// Forward: out = l0d*(l0h*(l0w*x[d0,h0,w0] + l1w*x[d0,h0,w1]) + l1h*(l0w*x[d0,h1,w0] + l1w*x[d0,h1,w1])) + l1d*(... d1 ...).
// Every product is computed, those with a zero weight included, so an inf or NaN in x spreads as it does through the op
// sequence.  A thread writes 4 consecutive outputs of a row (one float4 store when Wo % 4 == 0 and out is 16-byte aligned).
//
// Backward, a gather.  i0(o) never decreases as o grows (fp32 rounding is monotone), so the outputs that read input index i
// along an axis, those with i0(o) in {i-1, i}, form one range [b(i), e(i)).  A prep kernel tabulates per axis (i0, l1) of
// every output index and the range of every input index in the workspace, and one thread per input voxel sums
//   grad_x[d,h,w] = sum_od (sum_oh (sum_ow g[od,oh,ow]*ww) * wh) * wd
// with every sum started from 0 and taken in ascending o.  The weight of (o, i) along an axis is l0(o) if i0(o) == i, else
// l1(o); where i1(o) == i0(o) == i (the last index) the output adds both products, g*l0 first, then g*l1.  The order does
// not depend on the launch, so the bits are the same on every stream and run.  No atomics and no zero fill: every grad_x
// element is written once, 0 where no output reads it (downsampling).
#include "common.cuh"
#include "resize_taps.cuh"

namespace cspn {
namespace {

constexpr int kThreads = 256;
constexpr int kWCache = 12;     // W ranges up to this long keep their weights in registers (4x upsampling needs 8 or 9)

// ---- forward: grid (row quads of a slice, slices); a thread keeps its coordinates across the slices it visits -------------
__global__ void __launch_bounds__(kThreads)
resize_trilinear_fwd_kernel(const float* __restrict__ x, float* __restrict__ out, long long slices, Axis ad, Axis ah, Axis aw,
                            int quads, int vec) {
    const int Ho = ah.n_out, Wo = aw.n_out, H = ah.n_in, W = aw.n_in;
    const int q = blockIdx.x * kThreads + threadIdx.x;
    if (q >= ad.n_out * Ho * quads) return;
    const int ow0 = (q % quads) * 4, rest = q / quads, oh = rest % Ho, od = rest / Ho;
    const Tap td = tap_of(ad, od), th = tap_of(ah, oh);
    const int d1 = td.i0 + (td.i0 < ad.n_in - 1), h1 = th.i0 + (th.i0 < H - 1);
    const float l0d = __fsub_rn(1.f, td.l1), l0h = __fsub_rn(1.f, th.l1);
    int w0[4], w1[4];
    float l0w[4], l1w[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        const Tap tw = tap_of(aw, min(ow0 + k, Wo - 1));
        w0[k] = tw.i0;
        w1[k] = tw.i0 + (tw.i0 < W - 1);
        l1w[k] = tw.l1;
        l0w[k] = __fsub_rn(1.f, tw.l1);
    }
    const size_t vin = (size_t)ad.n_in * H * W, vout = (size_t)ad.n_out * Ho * Wo;
    const size_t r00 = ((size_t)td.i0 * H + th.i0) * W, r01 = ((size_t)td.i0 * H + h1) * W;
    const size_t r10 = ((size_t)d1 * H + th.i0) * W, r11 = ((size_t)d1 * H + h1) * W;
    const size_t o0 = ((size_t)od * Ho + oh) * Wo + ow0;
    for (long long bc = blockIdx.y; bc < slices; bc += gridDim.y) {
        const float* xs = x + (size_t)bc * vin;
        float v[4];
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            const float a00 = __fadd_rn(__fmul_rn(l0w[k], __ldg(xs + r00 + w0[k])), __fmul_rn(l1w[k], __ldg(xs + r00 + w1[k])));
            const float a01 = __fadd_rn(__fmul_rn(l0w[k], __ldg(xs + r01 + w0[k])), __fmul_rn(l1w[k], __ldg(xs + r01 + w1[k])));
            const float a10 = __fadd_rn(__fmul_rn(l0w[k], __ldg(xs + r10 + w0[k])), __fmul_rn(l1w[k], __ldg(xs + r10 + w1[k])));
            const float a11 = __fadd_rn(__fmul_rn(l0w[k], __ldg(xs + r11 + w0[k])), __fmul_rn(l1w[k], __ldg(xs + r11 + w1[k])));
            const float e0 = __fadd_rn(__fmul_rn(l0h, a00), __fmul_rn(th.l1, a01));
            const float e1 = __fadd_rn(__fmul_rn(l0h, a10), __fmul_rn(th.l1, a11));
            v[k] = __fadd_rn(__fmul_rn(l0d, e0), __fmul_rn(td.l1, e1));
        }
        float* o = out + (size_t)bc * vout + o0;
        if (vec) {
            *reinterpret_cast<float4*>(o) = make_float4(v[0], v[1], v[2], v[3]);
        } else {
#pragma unroll
            for (int k = 0; k < 4; ++k)
                if (ow0 + k < Wo) o[k] = v[k];
        }
    }
}

// ---- backward, gather: grid (input voxels of a slice, slices); one thread per input voxel -----------------------------------
__global__ void __launch_bounds__(kThreads)
resize_trilinear_bwd_kernel(const float* __restrict__ g, float* __restrict__ gx, const Tap* __restrict__ taps,
                            const Range* __restrict__ ranges, long long slices, int D, int H, int W, int Do, int Ho, int Wo) {
    const int v = blockIdx.x * kThreads + threadIdx.x;
    if (v >= D * H * W) return;
    const int w = v % W, rest = v / W, h = rest % H, d = rest / H;
    const Tap* td = taps;
    const Tap* th = taps + Do;
    const Tap* tw = taps + Do + Ho;
    const Range rd = ranges[d], rh = ranges[D + h], rw = ranges[D + H + w];
    const int nw = rw.e - rw.b;
    // the W weights, once for every row and slice: wa the first product's, wb the second's where the output adds two
    float wa[kWCache], wb[kWCache];
    unsigned twice = 0;
#pragma unroll
    for (int k = 0; k < kWCache; ++k) {
        const Tap t = k < nw && nw <= kWCache ? tw[rw.b + k] : Tap{-1, 0.f};
        wa[k] = t.i0 == w ? __fsub_rn(1.f, t.l1) : t.l1;
        wb[k] = t.l1;
        if (t.i0 == w && w == W - 1) twice |= 1u << k;
    }
    const size_t vin = (size_t)D * H * W, vout = (size_t)Do * Ho * Wo;
    for (long long bc = blockIdx.y; bc < slices; bc += gridDim.y) {
        const float* gs = g + (size_t)bc * vout;
        float acc_d = 0.f;
        for (int od = rd.b; od < rd.e; ++od) {
            float acc_h = 0.f;
            for (int oh = rh.b; oh < rh.e; ++oh) {
                const float* row = gs + ((size_t)od * Ho + oh) * Wo + rw.b;
                float acc_w = 0.f;
                if (nw <= kWCache) {
#pragma unroll
                    for (int k = 0; k < kWCache; ++k)
                        if (k < nw) {
                            const float gv = __ldg(row + k);
                            acc_w = __fadd_rn(acc_w, __fmul_rn(gv, wa[k]));
                            if (twice >> k & 1u) acc_w = __fadd_rn(acc_w, __fmul_rn(gv, wb[k]));
                        }
                } else {
                    for (int k = 0; k < nw; ++k) acc_w = add_tap(acc_w, __ldg(row + k), tw[rw.b + k], w, W);
                }
                acc_h = add_tap(acc_h, acc_w, th[oh], h, H);
            }
            acc_d = add_tap(acc_d, acc_h, td[od], d, D);
        }
        gx[(size_t)bc * vin + v] = acc_d;
    }
}

}  // namespace

int resize_trilinear_launchable(int D, int H, int W, int Do, int Ho, int Wo, const char** why) {
    if ((long long)D * H * W >= (1ll << 31)) { *why = "the input has >= 2^31 elements per (B*C) slice"; return 0; }
    if ((long long)Do * Ho * Wo >= (1ll << 31)) { *why = "the output has >= 2^31 elements per (B*C) slice"; return 0; }
    return 1;
}

size_t resize_trilinear_bwd_workspace_bytes(int D, int H, int W, int Do, int Ho, int Wo) {
    return ((size_t)Do + Ho + Wo) * sizeof(Tap) + ((size_t)D + H + W) * sizeof(Range);
}

int resize_trilinear_forward(const float* x, float* out, long long slices, int D, int H, int W, int Do, int Ho, int Wo,
                             int align_corners, int align_mode, cudaStream_t st, int* launches) {
    const int quads = (Wo + 3) / 4;
    const long long items = (long long)Do * Ho * quads;
    const int vec = Wo % 4 == 0 && (reinterpret_cast<uintptr_t>(out) & 15) == 0;
    resize_trilinear_fwd_kernel<<<dim3((unsigned)((items + kThreads - 1) / kThreads), slice_blocks(slices)), kThreads, 0, st>>>(
        x, out, slices, make_axis(D, Do, align_corners, align_mode), make_axis(H, Ho, align_corners, align_mode),
        make_axis(W, Wo, align_corners, align_mode), quads, vec);
    CSPN_CUDA_TRY(cudaGetLastError());
    *launches = 1;
    return CSPN_OK;
}

int resize_trilinear_backward(const float* grad_out, float* grad_x, long long slices, int D, int H, int W, int Do, int Ho,
                              int Wo, int align_corners, int align_mode, void* ws, cudaStream_t st, int* launches) {
    const Axis ad = make_axis(D, Do, align_corners, align_mode), ah = make_axis(H, Ho, align_corners, align_mode);
    const Axis aw = make_axis(W, Wo, align_corners, align_mode);
    const Tap* taps = static_cast<const Tap*>(ws);
    const Range* ranges = launch_resize_prep(ws, ad, ah, aw, st);
    CSPN_CUDA_TRY(cudaGetLastError());
    const long long vin = (long long)D * H * W;
    resize_trilinear_bwd_kernel<<<dim3((unsigned)((vin + kThreads - 1) / kThreads), slice_blocks(slices)), kThreads, 0, st>>>(
        grad_out, grad_x, taps, ranges, slices, D, H, W, Do, Ho, Wo);
    CSPN_CUDA_TRY(cudaGetLastError());
    *launches = 2;
    return CSPN_OK;
}

}  // namespace cspn
