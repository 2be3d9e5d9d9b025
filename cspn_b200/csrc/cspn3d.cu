// 3D CSPN (26 neighbours): prep (normalisation) + one 27-point stencil launch per iteration.
//
// Reference: call sites only -- /root/reference/cspn_paddle/demo.py:20-54; the Paddle op's
// source is not in the tree, so the arithmetic is the definition of SURVEY.md Appendix A.3
// (PARITY UNPINNED, see oracle/cspn_numpy.py).  Per-voxel state is 26 weights + kappa + value
// (112 B of input per voxel); with N = 12 and a 3D halo no on-chip temporal blocking fits an
// SM's 64K registers, so this path streams the normalised weights once per iteration from
// L2/HBM.  Volumes are processed in groups (grid z carries the volume index): one step launch covers the whole
// group, because a single volume's step is short enough that launch gaps and the grid's ramp / tail are a visible share;
// the group is capped so that the 27*D*H*W-float workspace per volume stays below kMaxWorkspace3d.
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

__global__ void __launch_bounds__(256)
step3d_kernel(const float* __restrict__ wk, const float* __restrict__ d0, const float* __restrict__ cur,
              float* __restrict__ dst, int C, int D, int H, int W) {
    const int x = blockIdx.x * blockDim.x + threadIdx.x;
    const int y = blockIdx.y * blockDim.y + threadIdx.y;
    const int z = blockIdx.z % D, c = blockIdx.z / D;   // c = volume * C + channel
    if (x >= W || y >= H) return;
    const size_t HW = (size_t)H * W, V = (size_t)D * HW;
    const size_t p = (size_t)z * HW + (size_t)y * W + x;
    wk += (size_t)(c / C) * 27 * V;
    const float* cc = cur + (size_t)c * V;
    float acc = __ldg(wk + 26 * V + p) * __ldg(d0 + (size_t)c * V + p);
#pragma unroll
    for (int k = 0; k < 26; ++k) {
        const int zz = z + off3_dz(k), yy = y + off3_dy(k), xx = x + off3_dx(k);
        const float dv = (zz >= 0 && zz < D && yy >= 0 && yy < H && xx >= 0 && xx < W)
                             ? __ldg(cc + (size_t)zz * HW + (size_t)yy * W + xx) : 0.f;
        acc = fmaf(__ldg(wk + k * V + p), dv, acc);
    }
    dst[(size_t)c * V + p] = acc;
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
__global__ void CSPN3D_BOUNDS
step3d_vec4_kernel(const float* __restrict__ wk, const float* __restrict__ d0, const float* __restrict__ cur,
                   float* __restrict__ dst, int C, int D, int H, int W) {
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
    const float4 kap = __ldg(reinterpret_cast<const float4*>(wk + 26 * V + p));
    const float4 dz0 = __ldg(reinterpret_cast<const float4*>(d0 + (size_t)c * V + p));
    float acc[4] = {kap.x * dz0.x, kap.y * dz0.y, kap.z * dz0.z, kap.w * dz0.w};
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
    *reinterpret_cast<float4*>(dst + (size_t)c * V + p) = make_float4(acc[0], acc[1], acc[2], acc[3]);
}

// 'paddle' normalisation straight from the RAW guidance (cspn_paddle/demo.py:24,47-52): the gate of tap k is
// |g_k(p)| / sum_j |g_j(p)| at the voxel's own location, so one step is  out(p) = (sum_k |g_k(p)| cur(p + off_k)) / (sum_k |g_k(p)|):
// ONE division per voxel instead of 26, no normalised-weight planes at all (no prep launch, no workspace for weights, 27
// instead of 29 planes read per step).  0 / 0 = NaN as with explicit gates.  The 26 guidance float4 of a thread are
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

#ifndef CSPN3D_PADDLE_BLOCKS
#define CSPN3D_PADDLE_BLOCKS 3
#endif
__global__ void __launch_bounds__(128, CSPN3D_PADDLE_BLOCKS)
step3d_paddle_vec4_kernel(const float* __restrict__ g, const float* __restrict__ cur, float* __restrict__ dst, int C, int D, int H,
                          int W) {
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
    *reinterpret_cast<float4*>(dst + (size_t)c * V + p) =
        make_float4(__fdiv_rn(acc[0], S[0]), __fdiv_rn(acc[1], S[1]), __fdiv_rn(acc[2], S[2]), __fdiv_rn(acc[3], S[3]));
}

// '26sum' / '26sum_abs' (gathered affinities + centre term, the cspn.py-style generalisation) straight from the RAW guidance,
// like the 'paddle' kernel above: a_k(p) = g_k(p + off_k) (zero outside the volume) is read where it lies -- an aligned float4
// of the shifted row plus, for dx = +-1, one neighbouring scalar (an L1 hit: the next thread's quad) -- S = sum |a_k|,
// w_k = a_k * (1 / S) (one division per voxel; where 1 / S overflows, i.e. S subnormal, the quotients are formed exactly),
// kappa = 1 - sum_k w_k from the products as the weight-plane path forms it from its quotients, out = kappa d0 + sum_k w_k
// cur(p + off_k).  No prep launch, no 27-plane workspace (1.65 GB for cfg4), 26 + 2 instead of 29 + 27/N planes per step.
#ifndef CSPN3D_GATHER_BLOCKS
#define CSPN3D_GATHER_BLOCKS 3
#endif
template <bool ABS>
__global__ void __launch_bounds__(128, CSPN3D_GATHER_BLOCKS)
step3d_gather_vec4_kernel(const float* __restrict__ g, const float* __restrict__ d0, const float* __restrict__ cur,
                          float* __restrict__ dst, int C, int D, int H, int W) {
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
    if (inv[0] > 8.0e37f || inv[1] > 8.0e37f || inv[2] > 8.0e37f || inv[3] > 8.0e37f) {   // cold: S subnormal, 1 / S overflowed
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            if (!(inv[j] > 8.0e37f)) continue;
            acc[j] = 0.f; s[j] = 0.f;
#pragma unroll
            for (int k = 0; k < 26; ++k) {
                const float av = j == 0 ? a[k].x : (j == 1 ? a[k].y : (j == 2 ? a[k].z : a[k].w));
                const float w = __fdiv_rn(av, S[j]);
                s[j] += w;
                acc[j] = fmaf(w, rows[off3_dz(k) + 1][off3_dy(k) + 1][1 + off3_dx(k) + j], acc[j]);
            }
        }
    }
    const float4 dz0 = __ldg(reinterpret_cast<const float4*>(d0 + (size_t)c * V + p));
    *reinterpret_cast<float4*>(dst + (size_t)c * V + p) =
        make_float4(fmaf(1.f - s[0], dz0.x, acc[0]), fmaf(1.f - s[1], dz0.y, acc[1]), fmaf(1.f - s[2], dz0.z, acc[2]),
                    fmaf(1.f - s[3], dz0.w, acc[3]));
}

}  // namespace

// Volumes per launch group: as many as keep the group's workspace under kMaxWorkspace3d (and gridDim.z legal).
constexpr size_t kMaxWorkspace3d = (size_t)4 << 30;
static int group3d(int B, int C, int D, int H, int W, int iters) {
    const size_t V = (size_t)D * H * W;
    const size_t per_vol = sizeof(float) * (27 * V + (iters > 1 ? (size_t)C * V : 0));
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
    return sizeof(float) * (size_t)group3d(B, C, D, H, W, iters) * (27 * V + (iters > 1 ? (size_t)C * V : 0));
}

int generic3d_forward(const float* guidance, const float* feat, float* out, int B, int C, int D, int H, int W,
                      int iters, int mode, void* ws, size_t ws_bytes, cudaStream_t stream, int* launches) {
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
        const dim3 grid((W / 4 + 31) / 32, (H + 3) / 4, D * C * B), block(32, 4);
        for (int it = 0; it < iters; ++it) {
            if (mode == 2) step3d_paddle_vec4_kernel<<<grid, block, 0, stream>>>(guidance, cur, dst, C, D, H, W);
            else if (mode == 1) step3d_gather_vec4_kernel<true><<<grid, block, 0, stream>>>(guidance, feat, cur, dst, C, D, H, W);
            else step3d_gather_vec4_kernel<false><<<grid, block, 0, stream>>>(guidance, feat, cur, dst, C, D, H, W);
            ++*launches;
            cur = dst;
            dst = (dst == out) ? tmp : out;
        }
        CSPN_CUDA_TRY(cudaGetLastError());
        return CSPN_OK;
    }
    const int G = group3d(B, C, D, H, W, iters);
    float* wk = static_cast<float*>(ws);          // [G][27][V]
    float* tmp = wk + (size_t)G * 27 * V;         // [G][C][V]
    const dim3 block(32, 8);
    const dim3 g2((W + 31) / 32, (H + 7) / 8);
    const bool vec4 = (W % 4 == 0) && ((reinterpret_cast<uintptr_t>(feat) | reinterpret_cast<uintptr_t>(out) |
                                          reinterpret_cast<uintptr_t>(ws)) % 16 == 0);
    for (int b0 = 0; b0 < B; b0 += G) {
        const int n = (B - b0 < G) ? B - b0 : G;  // volumes in this group
        const float* d0 = feat + (size_t)b0 * C * V;
        float* o = out + (size_t)b0 * C * V;
        prep3d_kernel<<<dim3(g2.x, g2.y, D * n), block, 0, stream>>>(guidance + (size_t)b0 * 26 * V, wk, D, H, W, mode);
        ++*launches;
        const float* cur = d0;
        float* dst = (iters & 1) ? o : tmp;
        for (int it = 0; it < iters; ++it) {
            if (vec4)
                step3d_vec4_kernel<<<dim3((W / 4 + 31) / 32, (H + 3) / 4, D * C * n), dim3(32, 4), 0, stream>>>(wk, d0, cur, dst, C, D, H, W);
            else
                step3d_kernel<<<dim3(g2.x, g2.y, D * C * n), block, 0, stream>>>(wk, d0, cur, dst, C, D, H, W);
            ++*launches;
            cur = dst;
            dst = (dst == o) ? tmp : o;
        }
    }
    CSPN_CUDA_TRY(cudaGetLastError());
    return CSPN_OK;
}

// ---- 3D backward (adjoint), one volume at a time; same scheme as cspn2d_bwd.cu with 26 taps ----------------------
// mode 0/1 ('26sum', '26sum_abs'): w_k = a_k / S with gathered a_k, kappa = 1 - sum w_k, c' = kappa d0:
//     Gkappa = sum_c Gc_c d0_c,  H_k = Gw_k - Gkappa,  T = sum_k H_k w_k,  dL/da_j = (H_j - sign(a_j) T) / S,
//     grad_g_j(p + off_j) = dL/da_j(p) [* sign(g_j) in abs mode],  grad_feat_c = kappa Gc_c + lambda_{0,c}.
// mode 2 ('paddle'): w_k(p) = |g_k(p)| / sum_j |g_j(p)| at the voxel's own location, no centre term:
//     H_k = Gw_k,  grad_g_j(p) = (H_j - T) / S * sign(g_j(p)),  grad_feat_c = lambda_{0,c}.
namespace {

__global__ void __launch_bounds__(256)
bwd3d_step_kernel(const float* __restrict__ wk, const float* __restrict__ d_t, const float* __restrict__ lam_in,
                  float* __restrict__ lam_out, float* __restrict__ Gw, float* __restrict__ Gc, int C, int D, int H, int W,
                  int first) {
    const int x = blockIdx.x * blockDim.x + threadIdx.x;
    const int y = blockIdx.y * blockDim.y + threadIdx.y;
    const int z = blockIdx.z;
    if (x >= W || y >= H) return;
    const size_t HW = (size_t)H * W, V = (size_t)D * HW;
    const size_t p = (size_t)z * HW + (size_t)y * W + x;
    for (int c = 0; c < C; ++c) {
        const float* li = lam_in + (size_t)c * V;
        const float* dt = d_t + (size_t)c * V;
        const float lp = __ldg(li + p);
        float acc = 0.f;
#pragma unroll
        for (int k = 0; k < 26; ++k) {
            const int zs = z - off3_dz(k), ys = y - off3_dy(k), xs = x - off3_dx(k);   // the voxel that reads me with tap k
            if (zs >= 0 && zs < D && ys >= 0 && ys < H && xs >= 0 && xs < W) {
                const size_t ps = (size_t)zs * HW + (size_t)ys * W + xs;
                acc = fmaf(__ldg(wk + k * V + ps), __ldg(li + ps), acc);
            }
            const int zn = z + off3_dz(k), yn = y + off3_dy(k), xn = x + off3_dx(k);
            float g = (first && c == 0) ? 0.f : Gw[k * V + p];
            if (zn >= 0 && zn < D && yn >= 0 && yn < H && xn >= 0 && xn < W)
                g = fmaf(lp, __ldg(dt + (size_t)zn * HW + (size_t)yn * W + xn), g);
            Gw[k * V + p] = g;
        }
        lam_out[(size_t)c * V + p] = acc;
        Gc[(size_t)c * V + p] = (first ? 0.f : Gc[(size_t)c * V + p]) + lp;
    }
}

__global__ void __launch_bounds__(256)
bwd3d_finalize_kernel(const float* __restrict__ g, const float* __restrict__ feat, const float* __restrict__ wk,
                      const float* __restrict__ Gw, const float* __restrict__ Gc, const float* __restrict__ lam0,
                      float* __restrict__ grad_g, float* __restrict__ grad_feat, int C, int D, int H, int W, int mode) {
    const int x = blockIdx.x * blockDim.x + threadIdx.x;
    const int y = blockIdx.y * blockDim.y + threadIdx.y;
    const int z = blockIdx.z;
    if (x >= W || y >= H) return;
    const size_t HW = (size_t)H * W, V = (size_t)D * HW;
    const size_t p = (size_t)z * HW + (size_t)y * W + x;
    const float kappa = __ldg(wk + 26 * V + p);
    float gkappa = 0.f;
    for (int c = 0; c < C; ++c) {
        const float gc = __ldg(Gc + (size_t)c * V + p);
        gkappa = fmaf(gc, __ldg(feat + (size_t)c * V + p), gkappa);
        if (grad_feat) grad_feat[(size_t)c * V + p] = fmaf(kappa, gc, __ldg(lam0 + (size_t)c * V + p));
    }
    if (!grad_g) return;
    if (mode == 2) gkappa = 0.f;   // no centre term
    float a[26], sg[26], S = 0.f;
#pragma unroll
    for (int k = 0; k < 26; ++k) {
        float v = 0.f;
        sg[k] = 1.f;
        if (mode == 2) {
            v = __ldg(g + k * V + p);
            sg[k] = signf(v);
            v = fabsf(v);
        } else {
            const int zz = z + off3_dz(k), yy = y + off3_dy(k), xx = x + off3_dx(k);
            if (zz >= 0 && zz < D && yy >= 0 && yy < H && xx >= 0 && xx < W) {
                v = __ldg(g + k * V + (size_t)zz * HW + (size_t)yy * W + xx);
                if (mode == 1) { sg[k] = signf(v); v = fabsf(v); }
            }
        }
        a[k] = v;
        S += fabsf(v);
    }
    float T = 0.f;
#pragma unroll
    for (int k = 0; k < 26; ++k) T = fmaf(__ldg(Gw + k * V + p) - gkappa, __fdiv_rn(a[k], S), T);
#pragma unroll
    for (int k = 0; k < 26; ++k) {
        const float ga = __fdiv_rn((__ldg(Gw + k * V + p) - gkappa) - signf(a[k]) * T, S) * sg[k];
        if (mode == 2) {
            grad_g[k * V + p] = ga;
        } else {
            const int zz = z + off3_dz(k), yy = y + off3_dy(k), xx = x + off3_dx(k);
            if (zz >= 0 && zz < D && yy >= 0 && yy < H && xx >= 0 && xx < W)
                grad_g[k * V + (size_t)zz * HW + (size_t)yy * W + xx] = ga;
        }
    }
}

}  // namespace

size_t bwd3d_workspace_bytes(int C, int D, int H, int W, int iters) {
    if (iters <= 0) return 0;
    const size_t V = (size_t)D * H * W, n = (size_t)C * V;
    // per volume: wk (27 planes) + d_1..d_{N-1} + lambda ping-pong + Gw (26 planes) + Gc
    return sizeof(float) * (27 * V + (size_t)(iters - 1) * n + 2 * n + 26 * V + n);
}

int bwd3d(const float* guidance, const float* feat, const float* grad_out, float* grad_guidance, float* grad_feat, int B, int C,
          int D, int H, int W, int iters, int mode, void* ws, size_t ws_bytes, cudaStream_t stream, int* launches) {
    const size_t V = (size_t)D * H * W, n = (size_t)C * V;
    if (grad_guidance) CSPN_CUDA_TRY(cudaMemsetAsync(grad_guidance, 0, (size_t)B * 26 * V * sizeof(float), stream));
    if (iters == 0) {
        if (grad_feat) CSPN_CUDA_TRY(cudaMemcpyAsync(grad_feat, grad_out, (size_t)B * n * sizeof(float), cudaMemcpyDeviceToDevice, stream));
        return CSPN_OK;
    }
    const size_t need = bwd3d_workspace_bytes(C, D, H, W, iters);
    if (!ws || ws_bytes < need) {
        set_error("3D backward needs %zu workspace bytes, got %zu", need, ws ? ws_bytes : (size_t)0);
        return CSPN_ERR_WORKSPACE;
    }
    if ((size_t)D * C > 65535) { set_error("3D backward: D*C exceeds gridDim.z"); return CSPN_ERR_UNSUPPORTED; }
    float* wk = static_cast<float*>(ws);
    float* Dt = wk + 27 * V;                                    // d_1 .. d_{N-1}
    float* lam[2] = {Dt + (size_t)(iters - 1) * n, Dt + (size_t)(iters - 1) * n + n};
    float* Gw = lam[1] + n;
    float* Gc = Gw + 26 * V;
    const dim3 block(32, 8);
    const dim3 g2((W + 31) / 32, (H + 7) / 8);
    for (int b = 0; b < B; ++b) {
        const float* gb = guidance + (size_t)b * 26 * V;
        const float* d0 = feat + (size_t)b * n;
        prep3d_kernel<<<dim3(g2.x, g2.y, D), block, 0, stream>>>(gb, wk, D, H, W, mode);
        ++*launches;
        for (int t = 0; t + 1 < iters; ++t) {
            step3d_kernel<<<dim3(g2.x, g2.y, D * C), block, 0, stream>>>(wk, d0, t == 0 ? d0 : Dt + (size_t)(t - 1) * n,
                                                                         Dt + (size_t)t * n, C, D, H, W);
            ++*launches;
        }
        const float* lam_in = grad_out + (size_t)b * n;
        for (int t = iters - 1; t >= 0; --t) {
            float* lam_out = lam[t & 1];
            bwd3d_step_kernel<<<dim3(g2.x, g2.y, D), block, 0, stream>>>(wk, t == 0 ? d0 : Dt + (size_t)(t - 1) * n, lam_in, lam_out,
                                                                         Gw, Gc, C, D, H, W, t == iters - 1);
            ++*launches;
            lam_in = lam_out;
        }
        bwd3d_finalize_kernel<<<dim3(g2.x, g2.y, D), block, 0, stream>>>(gb, d0, wk, Gw, Gc, lam_in,
                                                                         grad_guidance ? grad_guidance + (size_t)b * 26 * V : nullptr,
                                                                         grad_feat ? grad_feat + (size_t)b * n : nullptr, C, D, H, W, mode);
        ++*launches;
    }
    CSPN_CUDA_TRY(cudaGetLastError());
    return CSPN_OK;
}

}  // namespace cspn
