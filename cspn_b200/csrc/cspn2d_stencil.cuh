// The tile helpers of the launch-per-step K x K stencils that stage a plane with a halo in shared memory: the dilated
// propagation (cspn2d_dilated.cu, DESIGN.md section 4.22) and the dynamic propagation (cspn2d_dynamic.cu, section 4.23).
// Both replace with blend and load 4-pixel weights with ld4, so the replacement and the 4-pixel path's loads are one code.
#pragma once
#include <initializer_list>

#include "common.cuh"

namespace cspn {
namespace {

inline long long ceil_div(long long a, long long b) { return (a + b - 1) / b; }

__device__ __forceinline__ bool in_image(int y, int x, int H, int W) { return y >= 0 && y < H && x >= 0 && x < W; }

__device__ __forceinline__ float blend(float m, float s, float u) {
    return __fadd_rn(__fmul_rn(m, s), __fmul_rn(__fsub_rn(1.f, m), u));
}

__device__ __forceinline__ float4 ld4(const float* p) { return __ldg(reinterpret_cast<const float4*>(p)); }

// Stages rows y0 - h .. y0 + TH - 1 + h and columns x0 - h .. x0 + pitch - h - 1 of plane src into tile (the tile width
// plus 2h), zeros outside the image, with a CTA of TX x TY threads.  With a: each value is (1 - a(q)) * src(q) (the adjoint's
// mu = (1 - m) lambda).
template <int TX, int TY, int TH>
__device__ __forceinline__ void stage(float* tile, int pitch, const float* __restrict__ src, const float* __restrict__ a, int x0,
                                      int y0, int h, int H, int W) {
    const int n = (TH + 2 * h) * pitch;
    for (int i = threadIdx.y * TX + threadIdx.x; i < n; i += TX * TY) {
        const int gy = y0 - h + i / pitch, gx = x0 - h + i % pitch;
        float v = 0.f;
        if (in_image(gy, gx, H, W)) {
            const size_t q = (size_t)gy * W + gx;
            v = __ldg(src + q);
            if (a) v = __fmul_rn(__fsub_rn(1.f, __ldg(a + q)), v);
        }
        tile[i] = v;
    }
}

inline bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }

// The 4-pixel path: W % 4 == 0 and every plane it reads or writes with 16-byte accesses aligned
inline bool vec_ok(int W, std::initializer_list<const void*> ptrs) {
    if (W % 4) return false;
    for (const void* p : ptrs)
        if (p && !aligned16(p)) return false;
    return true;
}

}  // namespace
}  // namespace cspn
