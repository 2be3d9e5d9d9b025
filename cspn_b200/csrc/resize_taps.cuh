// The per-axis source coordinates of the Paddle module's resize_trilinear (DESIGN.md section 4.14), shared by the kernels
// that resample a volume: resize_trilinear.cu and disparity_regression.cu.  Both form every coordinate with tap_of, so both
// see the same bits, and both backward passes read the same per-axis tables, written by resize_trilinear_prep_kernel.
#pragma once
#include "common.cuh"

namespace cspn {
namespace {

constexpr int kPrepThreads = 256;

struct Axis {
    float r;
    int n_in, n_out;
    int half;                   // align_corners off with align_mode 0: the half-pixel rule
};

struct Tap {                    // an output index: its first source index and the weight of the second
    int i0;
    float l1;
};

struct Range {                  // an input index: the outputs [b, e) that read it
    int b, e;
};

__device__ __forceinline__ Tap tap_of(const Axis& a, int o) {
    const float fo = (float)o;
    const float s = a.half ? fmaxf(__fsub_rn(__fmul_rn(a.r, __fadd_rn(fo, 0.5f)), 0.5f), 0.f) : __fmul_rn(a.r, fo);
    const int i0 = min((int)s, a.n_in - 1);    // s < n_in for every size the entries take: the min only bounds the read
    return {i0, __fsub_rn(s, (float)i0)};
}

// the first output index whose i0 is >= i (n_out if none)
__device__ int first_output(const Axis& a, int i) {
    int lo = 0, hi = a.n_out;
    while (lo < hi) {
        const int m = lo + ((hi - lo) >> 1);
        if (tap_of(a, m).i0 >= i) hi = m;
        else lo = m + 1;
    }
    return lo;
}

// acc + the contribution of v through an output tap t to input index i of an axis of n_in
__device__ __forceinline__ float add_tap(float acc, float v, Tap t, int i, int n_in) {
    if (t.i0 != i) return __fadd_rn(acc, __fmul_rn(v, t.l1));
    acc = __fadd_rn(acc, __fmul_rn(v, __fsub_rn(1.f, t.l1)));
    return i == n_in - 1 ? __fadd_rn(acc, __fmul_rn(v, t.l1)) : acc;
}

// The taps of every output index and the range of every input index, D, H, W axes in turn: taps[Do + Ho + Wo], then
// ranges[D + H + W] (resize_trilinear_bwd_workspace_bytes() bytes).  One thread per entry.
__global__ void __launch_bounds__(kPrepThreads)
resize_trilinear_prep_kernel(Tap* __restrict__ taps, Range* __restrict__ ranges, Axis ad, Axis ah, Axis aw) {
    const long long e = (long long)blockIdx.x * kPrepThreads + threadIdx.x;
    const long long no = (long long)ad.n_out + ah.n_out + aw.n_out, ni = (long long)ad.n_in + ah.n_in + aw.n_in;
    if (e < no) {
        const int o = (int)(e < ad.n_out ? e : e < ad.n_out + ah.n_out ? e - ad.n_out : e - ad.n_out - ah.n_out);
        taps[e] = tap_of(e < ad.n_out ? ad : e < ad.n_out + ah.n_out ? ah : aw, o);
    } else if (e < no + ni) {
        const long long f = e - no;
        const Axis& a = f < ad.n_in ? ad : f < ad.n_in + ah.n_in ? ah : aw;
        const int i = (int)(f < ad.n_in ? f : f < ad.n_in + ah.n_in ? f - ad.n_in : f - ad.n_in - ah.n_in);
        ranges[f] = {first_output(a, i - 1), first_output(a, i + 1)};
    }
}

Axis make_axis(int n_in, int n_out, int align_corners, int align_mode) {
    Axis a;
    a.n_in = n_in;
    a.n_out = n_out;
    a.half = !align_corners && align_mode == 0;
    a.r = n_out == 1 ? 0.f : align_corners ? (float)(n_in - 1) / (float)(n_out - 1) : (float)n_in / (float)n_out;
    return a;
}

// Launches the prep kernel on the tables at the head of ws; returns the ranges
Range* launch_resize_prep(void* ws, const Axis& ad, const Axis& ah, const Axis& aw, cudaStream_t st) {
    Tap* taps = static_cast<Tap*>(ws);
    Range* ranges = reinterpret_cast<Range*>(taps + ((size_t)ad.n_out + ah.n_out + aw.n_out));
    const long long entries = (long long)ad.n_out + ah.n_out + aw.n_out + ad.n_in + ah.n_in + aw.n_in;
    resize_trilinear_prep_kernel<<<(unsigned)((entries + kPrepThreads - 1) / kPrepThreads), kPrepThreads, 0, st>>>(
        taps, ranges, ad, ah, aw);
    return ranges;
}

unsigned slice_blocks(long long slices) { return (unsigned)(slices < 65535 ? slices : 65535); }

}  // namespace
}  // namespace cspn
