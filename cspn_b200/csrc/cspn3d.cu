// 3D CSPN (26 neighbours), forward: prep (normalisation) + one 27-point stencil launch per iteration.  The 3x3x3
// backward runs on cspn3d_wide.cu's K x K x K kernels at R = 1.
//
// Reference: call sites only -- /root/reference/cspn_paddle/demo.py:20-54; the Paddle op's
// source is not in the tree, so the arithmetic is the definition of SURVEY.md Appendix A.3
// (PARITY UNPINNED, see oracle/cspn_numpy.py).  Per-voxel state is 26 weights + kappa + value
// (112 B of input per voxel); with N = 12 and a 3D halo no on-chip temporal blocking fits an
// SM's 64K registers, so this path streams the normalised weights once per iteration from
// L2/HBM.  Volumes are processed in groups (grid z carries the volume index): one step launch covers the whole
// group, because a single volume's step is short enough that launch gaps and the grid's ramp / tail are a visible share;
// the group is capped so that the 27*D*H*W-float workspace per volume stays below kMaxWorkspace3d.
//
// Fused gather (cspn3d_fwd_gather_f32, DESIGN.md section 4.6): the FAN flag of the step kernels stores each result also
// to the same element of every peer GPU's gather buffer (NVLink stores) and / or to one NVLS multicast address
// (multimem.st).  Only the last step, the one that writes `out`, runs it; the intermediate iterates never leave the GPU.
#include <cstdlib>

#include "common.cuh"

namespace cspn {

namespace {

// mode 0 '26sum', 1 '26sum_abs': gathered + centre term.  mode 2 'paddle': own location, no centre.
__global__ void __launch_bounds__(256)
prep3d_kernel(const float* __restrict__ g, float* __restrict__ wk, int D, int H, int W, int mode) {
    const int x = blockIdx.x * blockDim.x + threadIdx.x;
    const int y = blockIdx.y * blockDim.y + threadIdx.y;
    const int z = blockIdx.z % D, vol = blockIdx.z / D;
    if (x >= W || y >= H) return;
    const size_t HW = (size_t)H * W, V = (size_t)D * HW;
    const size_t p = (size_t)z * HW + (size_t)y * W + x;
    g += (size_t)vol * 26 * V;
    wk += (size_t)vol * 27 * V;
    float a[26], S = 0.f;
#pragma unroll
    for (int k = 0; k < 26; ++k) {
        float v;
        if (mode == 2) {
            v = fabsf(__ldg(g + k * V + p));
        } else {
            const int zz = z + off3_dz(k), yy = y + off3_dy(k), xx = x + off3_dx(k);
            v = 0.f;
            if (zz >= 0 && zz < D && yy >= 0 && yy < H && xx >= 0 && xx < W) {
                v = __ldg(g + k * V + (size_t)zz * HW + (size_t)yy * W + xx);
                if (mode == 1) v = fabsf(v);
            }
        }
        a[k] = v;
        S += fabsf(v);
    }
    float s = 0.f;
#pragma unroll
    for (int k = 0; k < 26; ++k) {
        const float w = __fdiv_rn(a[k], S);
        s += w;
        wk[k * V + p] = w;
    }
    wk[26 * V + p] = (mode == 2) ? 0.f : 1.f - s;
}

// FAN (every step kernel below): the result also goes to fan's destinations (the last step of a fused gather); fan is
// not read otherwise.  The two weight-plane steps add kappa d0 only where d0 is not null: 'paddle' has no centre term,
// and its kappa of 0 would still turn an inf or NaN of d0 into 0 * inf = NaN.
template <bool FAN = false>
__global__ void __launch_bounds__(256)
step3d_kernel(const float* __restrict__ wk, const float* __restrict__ d0, const float* __restrict__ cur,
              float* __restrict__ dst, int C, int D, int H, int W, const Fan fan) {
    const int x = blockIdx.x * blockDim.x + threadIdx.x;
    const int y = blockIdx.y * blockDim.y + threadIdx.y;
    const int z = blockIdx.z % D, c = blockIdx.z / D;   // c = volume * C + channel
    if (x >= W || y >= H) return;
    const size_t HW = (size_t)H * W, V = (size_t)D * HW;
    const size_t p = (size_t)z * HW + (size_t)y * W + x;
    wk += (size_t)(c / C) * 27 * V;
    const float* cc = cur + (size_t)c * V;
    float acc = d0 ? __ldg(wk + 26 * V + p) * __ldg(d0 + (size_t)c * V + p) : 0.f;
#pragma unroll
    for (int k = 0; k < 26; ++k) {
        const int zz = z + off3_dz(k), yy = y + off3_dy(k), xx = x + off3_dx(k);
        const float dv = (zz >= 0 && zz < D && yy >= 0 && yy < H && xx >= 0 && xx < W)
                             ? __ldg(cc + (size_t)zz * HW + (size_t)yy * W + xx) : 0.f;
        acc = fmaf(__ldg(wk + k * V + p), dv, acc);
    }
    const size_t o = (size_t)c * V + p;
    dst[o] = acc;
    if constexpr (FAN) fan_store(fan, o, acc);
}

// Vectorised step for W % 4 == 0: one thread produces 4 consecutive voxels of a row.  The 27 weight planes stream
// through as LDG.128 (they are the HBM traffic of this path: 108 B per voxel and step), the 9 neighbouring rows of the
// current volume are read as one aligned float4 plus two edge scalars each (L1/L2 hits).
// CSPN3D_MIN_BLOCKS: build-time knob for the next tuning round (python -m cspn_b200.build --define CSPN3D_MIN_BLOCKS=8
// caps the kernel at 64 registers -> 32 instead of 24 resident warps per SM); unset = ptxas' own choice (75 registers).
#ifdef CSPN3D_MIN_BLOCKS
#define CSPN3D_BOUNDS __launch_bounds__(128, CSPN3D_MIN_BLOCKS)
#else
#define CSPN3D_BOUNDS __launch_bounds__(128)
#endif
template <bool FAN = false>
__global__ void CSPN3D_BOUNDS
step3d_vec4_kernel(const float* __restrict__ wk, const float* __restrict__ d0, const float* __restrict__ cur,
                   float* __restrict__ dst, int C, int D, int H, int W, const Fan fan) {
    const int x = (blockIdx.x * blockDim.x + threadIdx.x) * 4;
    const int y = blockIdx.y * blockDim.y + threadIdx.y;
    const int z = blockIdx.z % D, c = blockIdx.z / D;   // c = volume * C + channel
    if (x >= W || y >= H) return;
    const size_t HW = (size_t)H * W, V = (size_t)D * HW;
    const size_t p = (size_t)z * HW + (size_t)y * W + x;
    wk += (size_t)(c / C) * 27 * V;
    const float* cc = cur + (size_t)c * V;
    // rows[dz+1][dy+1][0..5] = cur(z+dz, y+dy, x-1 .. x+4), zero outside the volume
    float rows[3][3][6];
#pragma unroll
    for (int dz = -1; dz <= 1; ++dz)
#pragma unroll
        for (int dy = -1; dy <= 1; ++dy) {
            const int zz = z + dz, yy = y + dy;
            float* r = rows[dz + 1][dy + 1];
            if (zz >= 0 && zz < D && yy >= 0 && yy < H) {
                const float* src = cc + (size_t)zz * HW + (size_t)yy * W + x;
                const float4 v = __ldg(reinterpret_cast<const float4*>(src));
                r[1] = v.x; r[2] = v.y; r[3] = v.z; r[4] = v.w;
                r[0] = x > 0 ? __ldg(src - 1) : 0.f;
                r[5] = x + 4 < W ? __ldg(src + 4) : 0.f;
            } else {
#pragma unroll
                for (int i = 0; i < 6; ++i) r[i] = 0.f;
            }
        }
    float acc[4] = {0.f, 0.f, 0.f, 0.f};
    if (d0) {
        const float4 kap = __ldg(reinterpret_cast<const float4*>(wk + 26 * V + p));
        const float4 dz0 = __ldg(reinterpret_cast<const float4*>(d0 + (size_t)c * V + p));
        acc[0] = kap.x * dz0.x; acc[1] = kap.y * dz0.y; acc[2] = kap.z * dz0.z; acc[3] = kap.w * dz0.w;
    }
#pragma unroll
    for (int k = 0; k < 26; ++k) {
        const float4 w = __ldg(reinterpret_cast<const float4*>(wk + k * V + p));
        const float* r = rows[off3_dz(k) + 1][off3_dy(k) + 1];
        const int o = 1 + off3_dx(k);
        acc[0] = fmaf(w.x, r[o], acc[0]);
        acc[1] = fmaf(w.y, r[o + 1], acc[1]);
        acc[2] = fmaf(w.z, r[o + 2], acc[2]);
        acc[3] = fmaf(w.w, r[o + 3], acc[3]);
    }
    const size_t o = (size_t)c * V + p;
    const float4 v = make_float4(acc[0], acc[1], acc[2], acc[3]);
    *reinterpret_cast<float4*>(dst + o) = v;
    if constexpr (FAN) fan_store(fan, o, v);
}

// 'paddle' normalisation straight from the RAW guidance (cspn_paddle/demo.py:24,47-52): the gate of tap k is
// |g_k(p)| / sum_j |g_j(p)| at the voxel's own location, so one step is  out(p) = (sum_k |g_k(p)| cur(p + off_k)) / (sum_k |g_k(p)|):
// ONE division per voxel instead of 26, no normalised-weight planes at all (no prep launch, no workspace for weights, 27
// instead of 29 planes read per step).  Where S is 0, subnormal, inf or NaN, or the sum overflowed or met an inf / NaN of
// cur (cold_paddle), a lane forms the 26 quotients |g_k| / S one by one instead: 0 / 0 = NaN, exact weights at a subnormal
// S, weights of 0 where S overflowed, as the weight-plane path has them.  The 26 guidance float4 of a thread are
// requested back to back before any arithmetic (CSPN3D_HOIST, default on): the kernel lives on loads in flight.
#ifndef CSPN3D_HOIST
#define CSPN3D_HOIST 1
#endif
__device__ __forceinline__ float4 ld_stream(const float* p) {
    float4 v;
#if CSPN3D_HOIST
    asm volatile("ld.global.nc.L1::no_allocate.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "l"(p));
#else
    v = __ldg(reinterpret_cast<const float4*>(p));
#endif
    return v;
}

// The quotient form of one voxel (z, y, x), the cold path of the two raw-guidance steps below: (sum_k w_k cur(p + off_k),
// sum_k w_k) with w_k = a_k / S formed one by one, as prep3d_kernel forms the weight planes (MODE 0 '26sum', 1 '26sum_abs':
// a_k = g_k(p + off_k), zero outside; 2 'paddle': a_k = |g_k(p)|).  The gates and the neighbours are read again (L1 / L2
// hits), and the function stays out of line, so that the hot loops of the callers keep nothing live for it.
template <int MODE>
__device__ __noinline__ float2 quotient_voxel(const float* __restrict__ g, const float* __restrict__ cc, float S, int z, int y,
                                              int x, int D, int H, int W) {
    const size_t HW = (size_t)H * W, V = (size_t)D * HW, p = (size_t)z * HW + (size_t)y * W + x;
    float acc = 0.f, s = 0.f;
#pragma unroll 1
    for (int k = 0; k < 26; ++k) {
        const int zz = z + off3_dz(k), yy = y + off3_dy(k), xx = x + off3_dx(k);
        const bool in = zz >= 0 && zz < D && yy >= 0 && yy < H && xx >= 0 && xx < W;
        const size_t q = (size_t)zz * HW + (size_t)yy * W + xx;
        float a = MODE == 2 ? fabsf(__ldg(g + k * V + p)) : (in ? __ldg(g + k * V + q) : 0.f);
        if (MODE == 1) a = fabsf(a);
        const float w = __fdiv_rn(a, S);
        s += w;
        acc = fmaf(w, in ? __ldg(cc + q) : 0.f, acc);
    }
    return make_float2(acc, s);
}

#ifndef CSPN3D_PADDLE_BLOCKS
#define CSPN3D_PADDLE_BLOCKS 3
#endif
template <bool FAN = false>
__global__ void __launch_bounds__(128, CSPN3D_PADDLE_BLOCKS)
step3d_paddle_vec4_kernel(const float* __restrict__ g, const float* __restrict__ cur, float* __restrict__ dst, int C, int D, int H,
                          int W, const Fan fan) {
    const int x = (blockIdx.x * blockDim.x + threadIdx.x) * 4;
    const int y = blockIdx.y * blockDim.y + threadIdx.y;
    const int z = blockIdx.z % D, c = blockIdx.z / D;   // c = volume * C + channel
    if (x >= W || y >= H) return;
    const size_t HW = (size_t)H * W, V = (size_t)D * HW;
    const size_t p = (size_t)z * HW + (size_t)y * W + x;
    g += (size_t)(c / C) * 26 * V;
    const float* cc = cur + (size_t)c * V;
    float4 w[26];
#pragma unroll
    for (int k = 0; k < 26; ++k) w[k] = ld_stream(g + k * V + p);
    float rows[3][3][6];
#pragma unroll
    for (int dz = -1; dz <= 1; ++dz)
#pragma unroll
        for (int dy = -1; dy <= 1; ++dy) {
            const int zz = z + dz, yy = y + dy;
            float* r = rows[dz + 1][dy + 1];
            if (zz >= 0 && zz < D && yy >= 0 && yy < H) {
                const float* src = cc + (size_t)zz * HW + (size_t)yy * W + x;
                const float4 v = __ldg(reinterpret_cast<const float4*>(src));
                r[1] = v.x; r[2] = v.y; r[3] = v.z; r[4] = v.w;
                r[0] = x > 0 ? __ldg(src - 1) : 0.f;
                r[5] = x + 4 < W ? __ldg(src + 4) : 0.f;
            } else {
#pragma unroll
                for (int i = 0; i < 6; ++i) r[i] = 0.f;
            }
        }
    float acc[4] = {0.f, 0.f, 0.f, 0.f}, S[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
    for (int k = 0; k < 26; ++k) {
        const float a0 = fabsf(w[k].x), a1 = fabsf(w[k].y), a2 = fabsf(w[k].z), a3 = fabsf(w[k].w);
        const float* r = rows[off3_dz(k) + 1][off3_dy(k) + 1];
        const int o = 1 + off3_dx(k);
        S[0] += a0; S[1] += a1; S[2] += a2; S[3] += a3;
        acc[0] = fmaf(a0, r[o], acc[0]);
        acc[1] = fmaf(a1, r[o + 1], acc[1]);
        acc[2] = fmaf(a2, r[o + 2], acc[2]);
        acc[3] = fmaf(a3, r[o + 3], acc[3]);
    }
#pragma unroll
    for (int j = 0; j < 4; ++j)
        acc[j] = cold_paddle(S[j], acc[j]) ? quotient_voxel<2>(g, cc, S[j], z, y, x + j, D, H, W).x : __fdiv_rn(acc[j], S[j]);
    const size_t o = (size_t)c * V + p;
    const float4 v = make_float4(acc[0], acc[1], acc[2], acc[3]);
    *reinterpret_cast<float4*>(dst + o) = v;
    if constexpr (FAN) fan_store(fan, o, v);
}

// '26sum' / '26sum_abs' (gathered affinities + centre term, the cspn.py-style generalisation) straight from the RAW guidance,
// like the 'paddle' kernel above: a_k(p) = g_k(p + off_k) (zero outside the volume) is read where it lies -- an aligned float4
// of the shifted row plus, for dx = +-1, one neighbouring scalar (an L1 hit: the next thread's quad) -- S = sum |a_k|,
// w_k = a_k * (1 / S) (one division per voxel; where 1 / S overflows, i.e. S subnormal, or d0 is +-inf, quotient_voxel forms them),
// kappa = 1 - sum_k w_k from the products as the weight-plane path forms it from its quotients, out = kappa d0 + sum_k w_k
// cur(p + off_k).  No prep launch, no 27-plane workspace (1.65 GB for cfg4), 26 + 2 instead of 29 + 27/N planes per step.
#ifndef CSPN3D_GATHER_BLOCKS
#define CSPN3D_GATHER_BLOCKS 3
#endif
template <bool ABS, bool FAN = false>
__global__ void __launch_bounds__(128, CSPN3D_GATHER_BLOCKS)
step3d_gather_vec4_kernel(const float* __restrict__ g, const float* __restrict__ d0, const float* __restrict__ cur,
                          float* __restrict__ dst, int C, int D, int H, int W, const Fan fan) {
    const int x = (blockIdx.x * blockDim.x + threadIdx.x) * 4;
    const int y = blockIdx.y * blockDim.y + threadIdx.y;
    const int z = blockIdx.z % D, c = blockIdx.z / D;   // c = volume * C + channel
    // no early exit: the x-neighbours of a shifted quad come from the neighbouring lanes (a warp is 32 consecutive quads of
    // one row), so every lane takes part in the shuffles; lanes outside the volume contribute the zero padding
    const bool active = x < W && y < H;
    const int lane = threadIdx.x;
    const size_t HW = (size_t)H * W, V = (size_t)D * HW;
    const size_t p = (size_t)z * HW + (size_t)y * W + x;
    g += (size_t)(c / C) * 26 * V;
    const float* cc = cur + (size_t)c * V;
    // all loads first, back to back (the kernel lives on loads in flight); the lane shuffles that complete the shifted quads after
    float4 a[26];
    float edge[26];
#pragma unroll
    for (int k = 0; k < 26; ++k) {
        const int zz = z + off3_dz(k), yy = y + off3_dy(k);
        const bool in = active && zz >= 0 && zz < D && yy >= 0 && yy < H;
        const float* src = g + k * V + (size_t)zz * HW + (size_t)yy * W + x;
        a[k] = in ? ld_stream(src) : make_float4(0.f, 0.f, 0.f, 0.f);
        edge[k] = 0.f;
        if (off3_dx(k) == 1 && lane == 31 && in && x + 4 < W) edge[k] = __ldg(src + 4);    // the warp's edge lanes: one scalar each
        if (off3_dx(k) == -1 && lane == 0 && in && x > 0) edge[k] = __ldg(src - 1);
    }
    float S[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
    for (int k = 0; k < 26; ++k) {
        const float4 q = a[k];
        float4 v = q;
        if (off3_dx(k) == 1) {           // elements x+1 .. x+4: the last one is the next lane's first
            const float e = __shfl_down_sync(0xffffffffu, q.x, 1);
            v = make_float4(q.y, q.z, q.w, lane == 31 ? edge[k] : e);
        } else if (off3_dx(k) == -1) {   // elements x-1 .. x+2
            const float e = __shfl_up_sync(0xffffffffu, q.w, 1);
            v = make_float4(lane == 0 ? edge[k] : e, q.x, q.y, q.z);
        }
        if (ABS) v = make_float4(fabsf(v.x), fabsf(v.y), fabsf(v.z), fabsf(v.w));
        a[k] = v;
        S[0] += fabsf(v.x); S[1] += fabsf(v.y); S[2] += fabsf(v.z); S[3] += fabsf(v.w);
    }
    if (!active) return;
    float rows[3][3][6];
#pragma unroll
    for (int dz = -1; dz <= 1; ++dz)
#pragma unroll
        for (int dy = -1; dy <= 1; ++dy) {
            const int zz = z + dz, yy = y + dy;
            float* r = rows[dz + 1][dy + 1];
            if (zz >= 0 && zz < D && yy >= 0 && yy < H) {
                const float* src = cc + (size_t)zz * HW + (size_t)yy * W + x;
                const float4 v = __ldg(reinterpret_cast<const float4*>(src));
                r[1] = v.x; r[2] = v.y; r[3] = v.z; r[4] = v.w;
                r[0] = x > 0 ? __ldg(src - 1) : 0.f;
                r[5] = x + 4 < W ? __ldg(src + 4) : 0.f;
            } else {
#pragma unroll
                for (int i = 0; i < 6; ++i) r[i] = 0.f;
            }
        }
    const float inv[4] = {__fdiv_rn(1.f, S[0]), __fdiv_rn(1.f, S[1]), __fdiv_rn(1.f, S[2]), __fdiv_rn(1.f, S[3])};
    float acc[4] = {0.f, 0.f, 0.f, 0.f}, s[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
    for (int k = 0; k < 26; ++k) {
        const float* r = rows[off3_dz(k) + 1][off3_dy(k) + 1];
        const int o = 1 + off3_dx(k);
        const float w0 = a[k].x * inv[0], w1 = a[k].y * inv[1], w2 = a[k].z * inv[2], w3 = a[k].w * inv[3];
        s[0] += w0; s[1] += w1; s[2] += w2; s[3] += w3;
        acc[0] = fmaf(w0, r[o], acc[0]);
        acc[1] = fmaf(w1, r[o + 1], acc[1]);
        acc[2] = fmaf(w2, r[o + 2], acc[2]);
        acc[3] = fmaf(w3, r[o + 3], acc[3]);
    }
    // cold: S subnormal (1 / S overflowed), or d0 = +-inf, where kappa d0 is NaN or inf depending on whether kappa is exactly
    // 0, so kappa must be 1 - sum_k a_k / S of the quotients (the products a_k * (1 / S) round differently)
    const float4 dz0 = __ldg(reinterpret_cast<const float4*>(d0 + (size_t)c * V + p));
    const float d0v[4] = {dz0.x, dz0.y, dz0.z, dz0.w};
#pragma unroll
    for (int j = 0; j < 4; ++j)
        if (inv[j] > 8.0e37f || fabsf(d0v[j]) == INFINITY) {
            const float2 q = quotient_voxel<ABS ? 1 : 0>(g, cc, S[j], z, y, x + j, D, H, W);
            acc[j] = q.x; s[j] = q.y;
        }
    const size_t o = (size_t)c * V + p;
    const float4 v = make_float4(fmaf(1.f - s[0], dz0.x, acc[0]), fmaf(1.f - s[1], dz0.y, acc[1]),
                                 fmaf(1.f - s[2], dz0.z, acc[2]), fmaf(1.f - s[3], dz0.w, acc[3]));
    *reinterpret_cast<float4*>(dst + o) = v;
    if constexpr (FAN) fan_store(fan, o, v);
}

// One step straight from the raw guidance (every volume in one launch); FAN: the last step of a fused gather
template <bool FAN>
void launch_raw_step(int mode, const float* g, const float* feat, const float* cur, float* dst, int nvol, int C, int D, int H,
                     int W, cudaStream_t s, const Fan& fan) {
    const dim3 grid((W / 4 + 31) / 32, (H + 3) / 4, D * C * nvol), block(32, 4);
    if (mode == 2) step3d_paddle_vec4_kernel<FAN><<<grid, block, 0, s>>>(g, cur, dst, C, D, H, W, fan);
    else if (mode == 1) step3d_gather_vec4_kernel<true, FAN><<<grid, block, 0, s>>>(g, feat, cur, dst, C, D, H, W, fan);
    else step3d_gather_vec4_kernel<false, FAN><<<grid, block, 0, s>>>(g, feat, cur, dst, C, D, H, W, fan);
}

// One step on the weight planes of a volume group
template <bool FAN>
void launch_plane_step(bool vec4, const float* wk, const float* d0, const float* cur, float* dst, int nvol, int C, int D, int H,
                       int W, cudaStream_t s, const Fan& fan) {
    if (vec4)
        step3d_vec4_kernel<FAN><<<dim3((W / 4 + 31) / 32, (H + 3) / 4, D * C * nvol), dim3(32, 4), 0, s>>>(wk, d0, cur, dst, C, D,
                                                                                                         H, W, fan);
    else
        step3d_kernel<FAN><<<dim3((W + 31) / 32, (H + 7) / 8, D * C * nvol), dim3(32, 8), 0, s>>>(wk, d0, cur, dst, C, D, H, W,
                                                                                                fan);
}

}  // namespace

// Volumes per launch group: as many as keep the group's workspace (`planes` weight planes per volume plus the ping-pong
// buffer) under kMaxWorkspace3d (and gridDim.z legal).  27 planes here, K^3 in cspn3d_wide.cu.
constexpr size_t kMaxWorkspace3d = (size_t)4 << 30;
int group3d(int B, int C, int D, int H, int W, int iters, int planes) {
    const size_t V = (size_t)D * H * W;
    const size_t per_vol = sizeof(float) * ((size_t)planes * V + (iters > 1 ? (size_t)C * V : 0));
    size_t cap = kMaxWorkspace3d;
    if (const char* e = getenv("CSPN_B200_MAX_WS3D_KB"))   // developer hook: tests force small / ragged groups
        if (atof(e) > 0) cap = (size_t)(atof(e) * 1024.0);
    size_t g = cap / per_vol;
    const size_t gz = 65535 / ((size_t)D * C);
    if (g > gz) g = gz;
    if (g > (size_t)B) g = B;
    return g < 1 ? 1 : (int)g;
}

size_t generic3d_workspace_bytes(int B, int C, int D, int H, int W, int iters) {
    if (iters <= 0) return 0;
    const size_t V = (size_t)D * H * W;
    return sizeof(float) * (size_t)group3d(B, C, D, H, W, iters, 27) * (27 * V + (iters > 1 ? (size_t)C * V : 0));
}

// fan (fused gather): destinations addressed like out, which the last step also writes; in the weight-plane route each
// is offset to the volume group as `out` is.
int generic3d_forward(const float* guidance, const float* feat, float* out, int B, int C, int D, int H, int W,
                      int iters, int mode, void* ws, size_t ws_bytes, cudaStream_t stream, int* launches, const Fan* fan) {
    const size_t V = (size_t)D * H * W;
    if (iters == 0) {
        CSPN_CUDA_TRY(cudaMemcpyAsync(out, feat, (size_t)B * C * V * sizeof(float), cudaMemcpyDeviceToDevice,
                                      stream));
        return CSPN_OK;
    }
    const size_t need = generic3d_workspace_bytes(B, C, D, H, W, iters);
    if (!ws || ws_bytes < need) {
        set_error("3D path needs %zu workspace bytes, got %zu", need, ws ? ws_bytes : (size_t)0);
        return CSPN_ERR_WORKSPACE;
    }
    if ((size_t)D * C > 65535 || D > 65535) {
        set_error("3D path: D*C=%zu exceeds gridDim.z", (size_t)D * C);
        return CSPN_ERR_UNSUPPORTED;
    }
    const bool vec4_all = (W % 4 == 0) && ((reinterpret_cast<uintptr_t>(feat) | reinterpret_cast<uintptr_t>(out) |
                                              reinterpret_cast<uintptr_t>(ws) | reinterpret_cast<uintptr_t>(guidance)) % 16 == 0);
    const char* raw_env = getenv("CSPN_B200_3D_PADDLE");     // developer hook: "planes" forces the prep + weight-plane path
    if (vec4_all && !(raw_env && raw_env[0] == 'p') && (size_t)D * C * B <= 65535 &&
        (iters == 1 || ws_bytes >= (size_t)B * C * V * sizeof(float))) {
        // gates straight from the raw guidance ('paddle': own location; '26sum[_abs]': gathered), every volume in one launch
        // per step; the workspace's first C*B*V floats are the ping-pong buffer
        float* tmp = static_cast<float*>(ws);
        const float* cur = feat;
        float* dst = (iters & 1) ? out : tmp;
        for (int it = 0; it < iters; ++it) {
            if (fan && it == iters - 1) launch_raw_step<true>(mode, guidance, feat, cur, dst, B, C, D, H, W, stream, *fan);
            else launch_raw_step<false>(mode, guidance, feat, cur, dst, B, C, D, H, W, stream, Fan{});
            ++*launches;
            cur = dst;
            dst = (dst == out) ? tmp : out;
        }
        CSPN_CUDA_TRY(cudaGetLastError());
        return CSPN_OK;
    }
    const int G = group3d(B, C, D, H, W, iters, 27);
    float* wk = static_cast<float*>(ws);          // [G][27][V]
    float* tmp = wk + (size_t)G * 27 * V;         // [G][C][V]
    const dim3 block(32, 8);
    const dim3 g2((W + 31) / 32, (H + 7) / 8);
    const bool vec4 = (W % 4 == 0) && ((reinterpret_cast<uintptr_t>(feat) | reinterpret_cast<uintptr_t>(out) |
                                          reinterpret_cast<uintptr_t>(ws)) % 16 == 0);
    for (int b0 = 0; b0 < B; b0 += G) {
        const int n = (B - b0 < G) ? B - b0 : G;  // volumes in this group
        const float* d0 = feat + (size_t)b0 * C * V;
        const float* centre = mode == 2 ? nullptr : d0;   // 'paddle': no kappa d0 term in the steps
        float* o = out + (size_t)b0 * C * V;
        prep3d_kernel<<<dim3(g2.x, g2.y, D * n), block, 0, stream>>>(guidance + (size_t)b0 * 26 * V, wk, D, H, W, mode);
        ++*launches;
        const float* cur = d0;
        float* dst = (iters & 1) ? o : tmp;
        for (int it = 0; it < iters; ++it) {
            if (fan && it == iters - 1)
                launch_plane_step<true>(vec4, wk, centre, cur, dst, n, C, D, H, W, stream, offset_fan(*fan, (size_t)b0 * C * V));
            else
                launch_plane_step<false>(vec4, wk, centre, cur, dst, n, C, D, H, W, stream, Fan{});
            ++*launches;
            cur = dst;
            dst = (dst == o) ? tmp : o;
        }
    }
    CSPN_CUDA_TRY(cudaGetLastError());
    return CSPN_OK;
}

}  // namespace cspn
