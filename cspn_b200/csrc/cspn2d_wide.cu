// 2D CSPN with a K x K affinity kernel, K = 2R+1 in {5, 7} (K*K-1 = 24 / 48 neighbours), forward and backward.
// The 3x3 operator keeps its own forward kernels (cspn2d_cluster.cu, cspn2d_generic.cu) and its cluster backward
// (cspn2d_bwd.cu); its fallback backward is the one here at K = 3, whose taps are off2_dy / off2_dx in the same order.
//
// Arithmetic: cspn2d_generic.cu with K*K-1 taps.  Tap k enumerates (t, l) over [0,K)^2 in raster order without the
// centre (R, R) and reads the source at (dy, dx) = (R-t, R-l) (oracle/cspn_numpy_k.py::offsets_2d):
//   a_k(p) = ghat_k(p + off_k) (0 outside),  w_k = a_k / sum_j |a_j|,  s = sum_k w_k,  m = sign(sparse)
//   folded: w'_k = (1-m) w_k,  kappa = (1-m)(1-s) + m,   d_{t+1} = kappa d0 + sum_k w'_k shift_k(d_t).
//
// Why not the cluster kernel's design: it keeps 8 weights per pixel in registers for the whole run.  24 or 48 weights
// per pixel do not fit (a KITTI image's 24 folded planes, ~41 MB, exceed the register file of the whole GPU), so this
// path stores the folded weights (K*K planes per image, the last one kappa) and streams them once per step:
//   prep    one launch per group of images: gather, normalise, fold the mask;
//   step    one launch per step and group (grid z = image*channel).  The CTA stages its tile of d_t with an R-pixel halo
//           in shared memory (zeros outside the image); each weight plane is read once per step, as LDG.128 when
//           W % 4 == 0 and the pointers are 16-byte aligned (4 pixels of a row per thread), else one pixel per thread.
//   groups  the launches cover the whole batch: one prep, then N steps.  (Splitting the batch into groups whose weight
//           planes fit the L2 measured slower; see group_size.)
// Backward, in the staged form of cspn2d_bwd.cu: prep, N-1 forward steps that keep d_1..d_{N-1}, N adjoint steps
//   lambda_t(q) = sum_k w'_k(q - off_k) lambda_{t+1}(q - off_k) (lambda_{t+1} tile + halo in shared memory), and one
//   gather-finalize kernel (Gw_k, Gc in registers, then the chain rule of cspn2d_bwd.cu with K*K-1 taps).
//
// 'paddle' (cspn_paddle/demo.py with dimNum = 2), K = 2R+1 in {3, 5, 7}, on the same launches:
//   w_k(p) = |g_k(p)| / sum_j |g_j(p)| at the pixel's own location,   d_{t+1} = sum_k w_k d_t(p + off_k)
// with no centre term and no sparse replacement.  Its prep (prepk_paddle_kernel) writes w_k and a zero kappa plane; the
// step kernels' PADDLE flag drops the kappa d0 term and the d0 load; the adjoint step is shared as it is; the gather's
// PADDLE flag applies the own-location chain rule (grad_g_j at p, grad_feat = lambda_0).  K = 3 runs here on every
// route: the cluster kernel keeps the folded 3x3 form only.
//
// Caller-supplied gates (fluid.layers.affinity_propagate itself, DESIGN.md section 4.11), K in {3, 5, 7}:
//   d_{t+1}(p) = sum_k g_k(p) d_t(p + off_k)   with the gates used as given (no |.|, no normalisation, no centre term).
// The RAW flag of the step and adjoint kernels reads the caller's gates [image][NT][H][W] (NT planes per image instead of
// the workspace's NP); there is no prep launch.  The gather's RAW mode writes Gw_k to the gate gradient at p and does
// not read the gates; the last adjoint step writes lambda_0 straight into the input gradient.
//
// Fused gather (cspn2d_{k,paddle,gates}_fwd_gather_f32, DESIGN.md section 4.6): the FAN flag of the two step kernels
// stores each result also to the same element of every peer GPU's gather buffer (NVLink stores) and / or to one NVLS
// multicast address (multimem.st).  Only the last step of a launch group, the one that writes `out`, runs it; the
// intermediate iterates never leave the GPU.
//
// Aggregation (CSPN++'s context-aware CSPN, DESIGN.md section 4.20), the normalised family at K in {3, 5, 7}:
//   out = sum_j sw_j * d_{s_j}.  The forward's aggregated steps run stepk_agg_*_kernel, whose epilogue adds sw_j * d to
// `out` (the accumulator); the backward recomputes d_1..d_N, writes the weight gradient and mu_N = sw_{T-1} * grad_out in
// agg_gradw_kernel, injects sw_j * grad_out into the adjoint at the aggregated steps (adjk_inject_kernel), and runs the
// gather above with mu_N as its last adjoint.
#include <cstdlib>
#include <cstring>

#include "common.cuh"

namespace cspn {

namespace {

template <int R>
struct Taps {
    static constexpr int K = 2 * R + 1;
    static constexpr int NT = K * K - 1;   // neighbours
    static constexpr int NP = K * K;       // planes per image in the workspace: w'_0..w'_{NT-1}, kappa
    __host__ __device__ static constexpr int idx(int k) { return k >= NT / 2 ? k + 1 : k; }
    __host__ __device__ static constexpr int dy(int k) { return R - idx(k) / K; }
    __host__ __device__ static constexpr int dx(int k) { return R - idx(k) % K; }
};

__device__ __forceinline__ bool inside(int y, int x, int H, int W) { return y >= 0 && y < H && x >= 0 && x < W; }

// ---- prep: prep2d_kernel with NT taps.  grid z = image of the group (pointers offset to the group) ----------------
// KEEP (keep-sparse mode, DESIGN.md section 4.13): m = 1[sparse > 0], and d0 [image][C][H][W] receives
// (1-m) blur + m sparse, which the step kernels' constant term kappa * d0 then reads in place of blur.
template <int R, bool KEEP>
__device__ __forceinline__ void prepk_body(const float* __restrict__ guidance, const float* __restrict__ sparse,
                                           float* __restrict__ wk, const float* __restrict__ blur, float* __restrict__ d0, int C,
                                           int H, int W, int gch, int norm_abs) {
    using T = Taps<R>;
    const int x = blockIdx.x * blockDim.x + threadIdx.x;
    const int y = blockIdx.y * blockDim.y + threadIdx.y;
    const int b = blockIdx.z;
    if (x >= W || y >= H) return;
    const size_t HW = (size_t)H * W;
    const float* g = guidance + (size_t)b * gch * HW;
    float a[T::NT], S = 0.f;
#pragma unroll
    for (int k = 0; k < T::NT; ++k) {
        const int yy = y + T::dy(k), xx = x + T::dx(k);
        float v = 0.f;
        if (inside(yy, xx, H, W)) {
            v = __ldg(g + k * HW + (size_t)yy * W + xx);
            if (norm_abs) v = fabsf(v);
        }
        a[k] = v;
        S += fabsf(v);
    }
    const size_t p = (size_t)y * W + x;
    float m, sv = 0.f;
    if constexpr (KEEP) {
        sv = __ldg(sparse + (size_t)b * HW + p);
        m = sv > 0.f ? 1.f : 0.f;             // NaN, 0 and negative samples are not samples
    } else {
        m = sparse ? signf(__ldg(sparse + (size_t)b * HW + p)) : 0.f;
    }
    const float om = 1.f - m;
    float s = 0.f;
    float* o = wk + (size_t)b * T::NP * HW + p;
#pragma unroll
    for (int k = 0; k < T::NT; ++k) {
        const float w = __fdiv_rn(a[k], S);   // IEEE: 0/0 -> NaN, x/inf -> 0, subnormal S divides exactly
        s += w;
        o[k * HW] = om * w;
    }
    o[T::NT * HW] = om * (1.f - s) + m;
    if constexpr (KEEP)
        for (int c = 0; c < C; ++c) {
            const size_t q = ((size_t)b * C + c) * HW + p;
            d0[q] = __fadd_rn(__fmul_rn(om, __ldg(blur + q)), __fmul_rn(m, sv));
        }
}

template <int R>
__global__ void __launch_bounds__(256)
prepk_kernel(const float* __restrict__ guidance, const float* __restrict__ sparse, float* __restrict__ wk, int H, int W,
             int gch, int norm_abs) {
    prepk_body<R, false>(guidance, sparse, wk, nullptr, nullptr, 1, H, W, gch, norm_abs);
}

// sparse non-null
template <int R>
__global__ void __launch_bounds__(256)
prepk_keep_kernel(const float* __restrict__ guidance, const float* __restrict__ sparse, const float* __restrict__ blur,
                  float* __restrict__ wk, float* __restrict__ d0, int C, int H, int W, int gch, int norm_abs) {
    prepk_body<R, true>(guidance, sparse, wk, blur, d0, C, H, W, gch, norm_abs);
}

// 'paddle' prep: w_k = |g_k(p)| / sum_j |g_j(p)|, kappa = 0.  guidance [image][NT][H][W]; grid z = image of the group
template <int R>
__global__ void __launch_bounds__(256)
prepk_paddle_kernel(const float* __restrict__ guidance, float* __restrict__ wk, int H, int W) {
    using T = Taps<R>;
    const int x = blockIdx.x * blockDim.x + threadIdx.x;
    const int y = blockIdx.y * blockDim.y + threadIdx.y;
    const int b = blockIdx.z;
    if (x >= W || y >= H) return;
    const size_t HW = (size_t)H * W, p = (size_t)y * W + x;
    const float* g = guidance + (size_t)b * T::NT * HW + p;
    float a[T::NT], S = 0.f;
#pragma unroll
    for (int k = 0; k < T::NT; ++k) {
        a[k] = fabsf(__ldg(g + k * HW));
        S += a[k];
    }
    float* o = wk + (size_t)b * T::NP * HW + p;
#pragma unroll
    for (int k = 0; k < T::NT; ++k) o[k * HW] = __fdiv_rn(a[k], S);   // IEEE: 0/0 -> NaN, x/inf -> 0, subnormal S exact
    o[T::NT * HW] = 0.f;
}

// ---- step, 4 pixels of a row per thread (W % 4 == 0, 16-byte aligned cur / d0 / dst / wk) -------------------------
// Tile 64 x 16 pixels per CTA of 16 x 16 threads.  The shared tile holds rows y0-R .. y0+15+R and columns x0-4 ..
// x0+67 as float4 (the halo is rounded up to 4 columns so every row of a thread's window is three aligned LDS.128).
// PADDLE: no kappa d0 term (d0 is not read).  RAW (with PADDLE): wk is the caller's gates, NT planes per image.
// FAN: the result also goes to fan's destinations (the last step of a fused gather); fan is not read otherwise.
constexpr int kVecTW = 64, kVecTH = 16;

// AGG (aggregation, DESIGN.md section 4.20; not with PADDLE, RAW or FAN): the step also adds lam * d_{t+1} to agg, the
// running sum (first: agg = lam * d_{t+1}, agg not read); lam is plane j of the step weights [image][nw][H][W]; a null dst
// stores no iterate (the last step).
template <int R, bool PADDLE, bool RAW, bool FAN, bool AGG>
__device__ __forceinline__ void stepk_vec_body(const float* __restrict__ wk, const float* __restrict__ d0,
                                               const float* __restrict__ cur, float* __restrict__ dst, int C, int H, int W,
                                               const Fan& fan, const float* __restrict__ lam, int nw, float* __restrict__ agg,
                                               int first) {
    using T = Taps<R>;
    constexpr int SH = kVecTH + 2 * R, SQ = kVecTW / 4 + 2;
    __shared__ float4 tile[SH][SQ];
    const int x0 = blockIdx.x * kVecTW, y0 = blockIdx.y * kVecTH, bc = blockIdx.z;
    const size_t HW = (size_t)H * W;
    const float* c = cur + (size_t)bc * HW;
    for (int i = threadIdx.y * 16 + threadIdx.x; i < SH * SQ; i += 256) {
        const int r = i / SQ, q = i % SQ;
        const int gy = y0 - R + r, gx = x0 - 4 + 4 * q;
        float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
        if (inside(gy, gx, H, W)) v = __ldg(reinterpret_cast<const float4*>(c + (size_t)gy * W + gx));   // W % 4 == 0
        tile[r][q] = v;
    }
    __syncthreads();
    const int tx = threadIdx.x, ty = threadIdx.y;
    const int x = x0 + 4 * tx, y = y0 + ty;
    if (x >= W || y >= H) return;
    const size_t p = (size_t)y * W + x;
    const float* w = wk + (size_t)(bc / C) * (RAW ? T::NT : T::NP) * HW + p;
    float acc0 = 0.f, acc1 = 0.f, acc2 = 0.f, acc3 = 0.f;
    if (!PADDLE) {
        const float4 kap = __ldg(reinterpret_cast<const float4*>(w + T::NT * HW));
        const float4 dd = __ldg(reinterpret_cast<const float4*>(d0 + (size_t)bc * HW + p));
        acc0 = kap.x * dd.x; acc1 = kap.y * dd.y; acc2 = kap.z * dd.z; acc3 = kap.w * dd.w;
    }
#pragma unroll
    for (int t = 0; t < T::K; ++t) {
        const int r = ty + R + (R - t);                      // tile row of source row y + dy, dy = R - t
        const float4 A = tile[r][tx], B = tile[r][tx + 1], Cq = tile[r][tx + 2];
        const float row[12] = {A.x, A.y, A.z, A.w, B.x, B.y, B.z, B.w, Cq.x, Cq.y, Cq.z, Cq.w};   // columns x-4 .. x+7
#pragma unroll
        for (int l = 0; l < T::K; ++l) {
            if (t == R && l == R) continue;
            const int k = t * T::K + l - (t * T::K + l > T::NT / 2 ? 1 : 0);
            const int dx = R - l;
            const float4 wv = __ldg(reinterpret_cast<const float4*>(w + k * HW));
            acc0 = fmaf(wv.x, row[4 + dx], acc0);
            acc1 = fmaf(wv.y, row[5 + dx], acc1);
            acc2 = fmaf(wv.z, row[6 + dx], acc2);
            acc3 = fmaf(wv.w, row[7 + dx], acc3);
        }
    }
    const size_t o = (size_t)bc * HW + p;
    const float4 v = make_float4(acc0, acc1, acc2, acc3);
    if constexpr (AGG) {
        if (dst) *reinterpret_cast<float4*>(dst + o) = v;
        const float4 l = __ldg(reinterpret_cast<const float4*>(lam + (size_t)(bc / C) * nw * HW + p));
        float4 a = make_float4(__fmul_rn(l.x, v.x), __fmul_rn(l.y, v.y), __fmul_rn(l.z, v.z), __fmul_rn(l.w, v.w));
        if (!first) {
            const float4 q = *reinterpret_cast<const float4*>(agg + o);
            a = make_float4(__fadd_rn(q.x, a.x), __fadd_rn(q.y, a.y), __fadd_rn(q.z, a.z), __fadd_rn(q.w, a.w));
        }
        *reinterpret_cast<float4*>(agg + o) = a;
        return;
    }
    *reinterpret_cast<float4*>(dst + o) = v;
    if constexpr (FAN) fan_store(fan, o, v);
}

template <int R, bool PADDLE = false, bool RAW = false, bool FAN = false>
__global__ void __launch_bounds__(256)
stepk_vec_kernel(const float* __restrict__ wk, const float* __restrict__ d0, const float* __restrict__ cur,
                 float* __restrict__ dst, int C, int H, int W, const Fan fan) {
    stepk_vec_body<R, PADDLE, RAW, FAN, false>(wk, d0, cur, dst, C, H, W, fan, nullptr, 0, nullptr, 0);
}

template <int R>
__global__ void __launch_bounds__(256)
stepk_agg_vec_kernel(const float* __restrict__ wk, const float* __restrict__ d0, const float* __restrict__ cur,
                     float* __restrict__ dst, const float* __restrict__ lam, int nw, float* __restrict__ agg, int first, int C,
                     int H, int W) {
    stepk_vec_body<R, false, false, false, true>(wk, d0, cur, dst, C, H, W, Fan{}, lam, nw, agg, first);
}

// ---- step / adjoint, one pixel per thread (any W, any alignment).  Tile 32 x 8 pixels + R halo --------------------
constexpr int kSclTW = 32, kSclTH = 8;

template <int R>
__device__ __forceinline__ void load_tile_scalar(float (*tile)[kSclTW + 2 * R], const float* __restrict__ src, int x0, int y0,
                                                 int H, int W) {
    constexpr int SH = kSclTH + 2 * R, SW = kSclTW + 2 * R;
    for (int i = threadIdx.y * kSclTW + threadIdx.x; i < SH * SW; i += kSclTW * kSclTH) {
        const int r = i / SW, q = i % SW;
        const int gy = y0 - R + r, gx = x0 - R + q;
        tile[r][q] = inside(gy, gx, H, W) ? __ldg(src + (size_t)gy * W + gx) : 0.f;
    }
}

// AGG: as in stepk_vec_body
template <int R, bool PADDLE, bool RAW, bool FAN, bool AGG>
__device__ __forceinline__ void stepk_scalar_body(const float* __restrict__ wk, const float* __restrict__ d0,
                                                  const float* __restrict__ cur, float* __restrict__ dst, int C, int H, int W,
                                                  const Fan& fan, const float* __restrict__ lam, int nw, float* __restrict__ agg,
                                                  int first) {
    using T = Taps<R>;
    __shared__ float tile[kSclTH + 2 * R][kSclTW + 2 * R];
    const int x0 = blockIdx.x * kSclTW, y0 = blockIdx.y * kSclTH, bc = blockIdx.z;
    const size_t HW = (size_t)H * W;
    load_tile_scalar<R>(tile, cur + (size_t)bc * HW, x0, y0, H, W);
    __syncthreads();
    const int tx = threadIdx.x, ty = threadIdx.y, x = x0 + tx, y = y0 + ty;
    if (x >= W || y >= H) return;
    const size_t p = (size_t)y * W + x;
    const float* w = wk + (size_t)(bc / C) * (RAW ? T::NT : T::NP) * HW + p;
    float acc = PADDLE ? 0.f : __ldg(w + T::NT * HW) * __ldg(d0 + (size_t)bc * HW + p);
#pragma unroll
    for (int k = 0; k < T::NT; ++k) acc = fmaf(__ldg(w + k * HW), tile[ty + R + T::dy(k)][tx + R + T::dx(k)], acc);
    const size_t o = (size_t)bc * HW + p;
    if constexpr (AGG) {
        if (dst) dst[o] = acc;
        const float a = __fmul_rn(__ldg(lam + (size_t)(bc / C) * nw * HW + p), acc);
        agg[o] = first ? a : __fadd_rn(agg[o], a);
        return;
    }
    dst[o] = acc;
    if constexpr (FAN) fan_store(fan, o, acc);
}

template <int R, bool PADDLE = false, bool RAW = false, bool FAN = false>
__global__ void __launch_bounds__(256)
stepk_scalar_kernel(const float* __restrict__ wk, const float* __restrict__ d0, const float* __restrict__ cur,
                    float* __restrict__ dst, int C, int H, int W, const Fan fan) {
    stepk_scalar_body<R, PADDLE, RAW, FAN, false>(wk, d0, cur, dst, C, H, W, fan, nullptr, 0, nullptr, 0);
}

template <int R>
__global__ void __launch_bounds__(256)
stepk_agg_scalar_kernel(const float* __restrict__ wk, const float* __restrict__ d0, const float* __restrict__ cur,
                        float* __restrict__ dst, const float* __restrict__ lam, int nw, float* __restrict__ agg, int first, int C,
                        int H, int W) {
    stepk_scalar_body<R, false, false, false, true>(wk, d0, cur, dst, C, H, W, Fan{}, lam, nw, agg, first);
}

// lambda_t(q) = sum_k w'_k(q - off_k) lambda_{t+1}(q - off_k): the transposed stencil, source pixels inside the image only.
// RAW: wk is the caller's gates, NT planes per image.
// INJ (aggregation backward, mu_t of DESIGN.md section 4.20): then lam_out = lam_out + sw * grad_out, sw plane j of the step
// weights [image][nw][H][W], each operation rounded on its own.
template <int R, bool RAW, bool INJ>
__device__ __forceinline__ void adjk_body(const float* __restrict__ wk, const float* __restrict__ lam_in, float* __restrict__ lam_out,
                                          int C, int H, int W, const float* __restrict__ sw, int nw,
                                          const float* __restrict__ grad_out) {
    using T = Taps<R>;
    __shared__ float tile[kSclTH + 2 * R][kSclTW + 2 * R];
    const int x0 = blockIdx.x * kSclTW, y0 = blockIdx.y * kSclTH, bc = blockIdx.z;
    const size_t HW = (size_t)H * W;
    load_tile_scalar<R>(tile, lam_in + (size_t)bc * HW, x0, y0, H, W);
    __syncthreads();
    const int tx = threadIdx.x, ty = threadIdx.y, x = x0 + tx, y = y0 + ty;
    if (x >= W || y >= H) return;
    const float* w = wk + (size_t)(bc / C) * (RAW ? T::NT : T::NP) * HW;
    float acc = 0.f;
#pragma unroll
    for (int k = 0; k < T::NT; ++k) {
        const int ys = y - T::dy(k), xs = x - T::dx(k);
        if (inside(ys, xs, H, W))
            acc = fmaf(__ldg(w + k * HW + (size_t)ys * W + xs), tile[ty + R - T::dy(k)][tx + R - T::dx(k)], acc);
    }
    const size_t p = (size_t)y * W + x;
    if constexpr (INJ)
        acc = __fadd_rn(acc, __fmul_rn(__ldg(sw + (size_t)(bc / C) * nw * HW + p), __ldg(grad_out + (size_t)bc * HW + p)));
    lam_out[(size_t)bc * HW + p] = acc;
}

template <int R, bool RAW = false>
__global__ void __launch_bounds__(256)
adjk_kernel(const float* __restrict__ wk, const float* __restrict__ lam_in, float* __restrict__ lam_out, int C, int H,
            int W) {
    adjk_body<R, RAW, false>(wk, lam_in, lam_out, C, H, W, nullptr, 0, nullptr);
}

template <int R>
__global__ void __launch_bounds__(256)
adjk_inject_kernel(const float* __restrict__ wk, const float* __restrict__ lam_in, float* __restrict__ lam_out,
                   const float* __restrict__ sw, int nw, const float* __restrict__ grad_out, int C, int H, int W) {
    adjk_body<R, false, true>(wk, lam_in, lam_out, C, H, W, sw, nw, grad_out);
}

// The step-weight gradient and the last adjoint of the aggregation (DESIGN.md section 4.20), one pixel per thread, grid
// z = image of the group: for the steps s_j, j = j0 .. j0+ns-1, of `sel`
//   grad_sw[j](p) = sum_c grad_out[c](p) * d_{s_j}[c](p)     (c ascending from the first term; skipped when grad_sw is null)
// and, when mu is non-null, mu[c](p) = sw[nw-1](p) * grad_out[c](p) = mu_N.  d_s is plane s-1 of `iters` (planes n floats
// apart); every pointer is offset to the group's first image.
constexpr int kAggStepsPerLaunch = 64;
struct StepSel {
    int s[kAggStepsPerLaunch];
};

__global__ void __launch_bounds__(256)
agg_gradw_kernel(const float* __restrict__ grad_out, const float* __restrict__ iters, long long n, const float* __restrict__ sw,
                 float* __restrict__ grad_sw, float* __restrict__ mu, const StepSel sel, int j0, int ns, int nw, int C,
                 long long HW) {
    const long long p = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const int b = blockIdx.z;
    if (p >= HW) return;
    const float* g = grad_out + (size_t)b * C * HW + p;
    if (grad_sw)
        for (int j = 0; j < ns; ++j) {
            const float* d = iters + (size_t)(sel.s[j] - 1) * n + (size_t)b * C * HW + p;
            float a = __fmul_rn(__ldg(g), __ldg(d));
            for (int c = 1; c < C; ++c) a = __fadd_rn(a, __fmul_rn(__ldg(g + c * HW), __ldg(d + c * HW)));
            grad_sw[((size_t)b * nw + j0 + j) * HW + p] = a;
        }
    if (mu) {
        const float l = __ldg(sw + ((size_t)b * nw + nw - 1) * HW + p);
        for (int c = 0; c < C; ++c) mu[(size_t)b * C * HW + c * HW + p] = __fmul_rn(l, __ldg(g + c * HW));
    }
}

// Gw_k(p) = sum_t lambda_{t+1}(p) d_t(p + off_k) with d_t staged tile by tile, Gc = sum_t lambda_{t+1}; then the finalize
// arithmetic of cspn2d_bwd.cu.  steps[t] = d_{t+1}, lam[t] = lambda_t (planes n floats apart), lambda_N = grad_out.
// grid z = image of the group; every pointer is offset to the group's first image.
// PADDLE (sparse null, gch = NT): the own-location chain rule of cspn3d_wide.cu's fin3k_kernel mode 2 -- no centre term,
// grad_g_j lands at p, grad_blur = lambda_0.
// RAW (with PADDLE, grad_blur null): the gates are the caller's, so grad_g_k(p) = Gw_k(p); guidance and wk are not read.
// KEEP (keep-sparse mode, sparse non-null): m = 1[sparse > 0], grad_blur's coefficient is (1-m)(1-s) = kappa - m, and
// grad_sparse (may be null) receives m * sum_c Gc_c, the channels summed in order.
template <int R, bool PADDLE, bool RAW, bool KEEP>
__device__ __forceinline__ void gatherk_body(const float* __restrict__ guidance, const float* __restrict__ blur,
                                             const float* __restrict__ sparse, const float* __restrict__ wk,
                                             const float* __restrict__ steps, const float* __restrict__ lam,
                                             const float* __restrict__ grad_out, float* __restrict__ grad_guidance,
                                             float* __restrict__ grad_blur, float* __restrict__ grad_sparse, long long n, int N,
                                             int C, int H, int W, int gch, int norm_abs) {
    using T = Taps<R>;
    __shared__ float tile[kSclTH + 2 * R][kSclTW + 2 * R];
    const int x0 = blockIdx.x * kSclTW, y0 = blockIdx.y * kSclTH, b = blockIdx.z;
    const int tx = threadIdx.x, ty = threadIdx.y, x = x0 + tx, y = y0 + ty;
    const bool in = x < W && y < H;
    const size_t HW = (size_t)H * W, p = in ? (size_t)y * W + x : 0;
    float gw[T::NT];
#pragma unroll
    for (int k = 0; k < T::NT; ++k) gw[k] = 0.f;
    const float kappa = in && !PADDLE ? __ldg(wk + ((size_t)b * T::NP + T::NT) * HW + p) : 0.f;
    [[maybe_unused]] float m_keep = 0.f, gsum = 0.f;
    if constexpr (KEEP) m_keep = in && __ldg(sparse + (size_t)b * HW + p) > 0.f ? 1.f : 0.f;
    const float cblur = KEEP ? kappa - m_keep : kappa;
    float gkappa = 0.f;
    for (int c = 0; c < C; ++c) {
        const size_t plane = ((size_t)b * C + c) * HW;
        float gc = 0.f;
        for (int t = 0; t < N; ++t) {
            __syncthreads();
            load_tile_scalar<R>(tile, (t == 0 ? blur : steps + (size_t)(t - 1) * n) + plane, x0, y0, H, W);
            __syncthreads();
            if (!in) continue;
            const float lp = __ldg((t == N - 1 ? grad_out : lam + (size_t)(t + 1) * n) + plane + p);
            gc += lp;
#pragma unroll
            for (int k = 0; k < T::NT; ++k)   // taps outside the image take no gradient (they read the zero padding)
                if (inside(y + T::dy(k), x + T::dx(k), H, W))
                    gw[k] = fmaf(lp, tile[ty + R + T::dy(k)][tx + R + T::dx(k)], gw[k]);
        }
        if (!in) continue;
        if (PADDLE) {
            if (grad_blur) grad_blur[plane + p] = __ldg(lam + plane + p);
            continue;
        }
        gkappa = fmaf(gc, __ldg(blur + plane + p), gkappa);
        if (grad_blur) grad_blur[plane + p] = fmaf(cblur, gc, __ldg(lam + plane + p));   // lam[0] = lambda_0
        if constexpr (KEEP) gsum += gc;
    }
    if constexpr (KEEP)
        if (in && grad_sparse) grad_sparse[(size_t)b * HW + p] = m_keep * gsum;
    if (!in || !grad_guidance) return;
    if (RAW) {
#pragma unroll
        for (int k = 0; k < T::NT; ++k) grad_guidance[((size_t)b * T::NT + k) * HW + p] = gw[k];
        return;
    }
    const float* g = guidance + (size_t)b * gch * HW;
    if (PADDLE) {
        float S = 0.f;
#pragma unroll
        for (int k = 0; k < T::NT; ++k) S += fabsf(__ldg(g + k * HW + p));
        float Tsum = 0.f;
#pragma unroll
        for (int k = 0; k < T::NT; ++k) Tsum = fmaf(gw[k], __fdiv_rn(fabsf(__ldg(g + k * HW + p)), S), Tsum);
#pragma unroll
        for (int k = 0; k < T::NT; ++k) {   // d|g|/dg = sign(g), 0 at 0 like torch.abs
            const float v = __ldg(g + k * HW + p);
            grad_guidance[((size_t)b * gch + k) * HW + p] = __fdiv_rn(gw[k] - signf(fabsf(v)) * Tsum, S) * signf(v);
        }
        return;
    }
    float a[T::NT], S = 0.f;
#pragma unroll
    for (int k = 0; k < T::NT; ++k) {
        const int yy = y + T::dy(k), xx = x + T::dx(k);
        float v = 0.f;
        if (inside(yy, xx, H, W)) {
            v = __ldg(g + k * HW + (size_t)yy * W + xx);
            if (norm_abs) v = fabsf(v);
        }
        a[k] = v;
        S += fabsf(v);
    }
    const float m = KEEP ? m_keep : sparse ? signf(__ldg(sparse + (size_t)b * HW + p)) : 0.f;
    const float om = 1.f - m;
    float Tsum = 0.f;
#pragma unroll
    for (int k = 0; k < T::NT; ++k) {
        gw[k] = om * (gw[k] - gkappa);                          // H_k = dL/dw_k
        Tsum = fmaf(gw[k], __fdiv_rn(a[k], S), Tsum);
    }
#pragma unroll
    for (int k = 0; k < T::NT; ++k) {
        const int yy = y + T::dy(k), xx = x + T::dx(k);
        if (inside(yy, xx, H, W)) {
            const size_t q = (size_t)yy * W + xx;
            const float ga = __fdiv_rn(gw[k] - signf(a[k]) * Tsum, S);
            // d|g|/dg = sign(g) (0 at 0, like torch.abs) in the _abs norm
            const float sg = norm_abs ? signf(__ldg(g + k * HW + q)) : 1.f;
            grad_guidance[((size_t)b * gch + k) * HW + q] = ga * sg;
        }
    }
}

template <int R, bool PADDLE = false, bool RAW = false>
__global__ void __launch_bounds__(256)
gatherk_kernel(const float* __restrict__ guidance, const float* __restrict__ blur, const float* __restrict__ sparse,
               const float* __restrict__ wk, const float* __restrict__ steps, const float* __restrict__ lam,
               const float* __restrict__ grad_out, float* __restrict__ grad_guidance, float* __restrict__ grad_blur,
               long long n, int N, int C, int H, int W, int gch, int norm_abs) {
    gatherk_body<R, PADDLE, RAW, false>(guidance, blur, sparse, wk, steps, lam, grad_out, grad_guidance, grad_blur, nullptr, n, N,
                                        C, H, W, gch, norm_abs);
}

template <int R>
__global__ void __launch_bounds__(256)
gatherk_keep_kernel(const float* __restrict__ guidance, const float* __restrict__ blur, const float* __restrict__ sparse,
                    const float* __restrict__ wk, const float* __restrict__ steps, const float* __restrict__ lam,
                    const float* __restrict__ grad_out, float* __restrict__ grad_guidance, float* __restrict__ grad_blur,
                    float* __restrict__ grad_sparse, long long n, int N, int C, int H, int W, int gch, int norm_abs) {
    gatherk_body<R, false, false, true>(guidance, blur, sparse, wk, steps, lam, grad_out, grad_guidance, grad_blur, grad_sparse, n,
                                        N, C, H, W, gch, norm_abs);
}

bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }

// Images per launch group: the whole batch.  Groups sized so that their weight planes fit the L2 (steps 2..N reading
// the weights from L2 instead of HBM) measured slower than one group on an H100 at 3 of the 4 shapes of
// tools/time_kxk.py (DESIGN.md section 4.8), so they are not used.  CSPN_B200_KXK_GROUP=<images> splits the batch
// (developer hook: the tests check that an image's bits do not depend on its group; time_kxk.py compares the two).
int group_size(int B) {
    if (const char* e = getenv("CSPN_B200_KXK_GROUP")) {
        const int v = atoi(e);
        if (v > 0) return v < B ? v : B;
    }
    return B;
}

template <int R, bool PADDLE>
void launch_prep(const float* guidance, const float* sparse, float* wk, int nimg, int H, int W, int gch, int norm_abs,
                 cudaStream_t s) {
    const dim3 grid((W + 31) / 32, (H + 7) / 8, nimg), block(32, 8);
    if constexpr (PADDLE) prepk_paddle_kernel<R><<<grid, block, 0, s>>>(guidance, wk, H, W);
    else prepk_kernel<R><<<grid, block, 0, s>>>(guidance, sparse, wk, H, W, gch, norm_abs);
}

// fan non-null: the FAN instantiation, which also stores the result to fan's destinations
template <int R, bool PADDLE, bool RAW = false>
void launch_step(bool vec, const float* wk, const float* d0, const float* cur, float* dst, int nbc, int C, int H, int W,
                 cudaStream_t s, const Fan* fan = nullptr) {
    const dim3 vgrid((W + kVecTW - 1) / kVecTW, (H + kVecTH - 1) / kVecTH, nbc), vblock(16, 16);
    const dim3 sgrid((W + kSclTW - 1) / kSclTW, (H + kSclTH - 1) / kSclTH, nbc), sblock(kSclTW, kSclTH);
    if (fan) {
        if (vec) stepk_vec_kernel<R, PADDLE, RAW, true><<<vgrid, vblock, 0, s>>>(wk, d0, cur, dst, C, H, W, *fan);
        else stepk_scalar_kernel<R, PADDLE, RAW, true><<<sgrid, sblock, 0, s>>>(wk, d0, cur, dst, C, H, W, *fan);
        return;
    }
    if (vec) stepk_vec_kernel<R, PADDLE, RAW><<<vgrid, vblock, 0, s>>>(wk, d0, cur, dst, C, H, W, Fan{});
    else stepk_scalar_kernel<R, PADDLE, RAW><<<sgrid, sblock, 0, s>>>(wk, d0, cur, dst, C, H, W, Fan{});
}

// RAW: the caller's gates (p.guidance, NT planes per image) are the weight planes; the workspace holds only the
// ping-pong buffer.  fan (fused gather): destinations addressed like p.out, which the last step of every launch group
// also writes, each offset to the group as `out` is.
template <int R, bool PADDLE, bool RAW = false>
int forward_k(const Problem2D& p, void* ws, cudaStream_t stream, int* launches, const Fan* fan = nullptr) {
    constexpr int NPL = RAW ? Taps<R>::NT : Taps<R>::NP;   // weight planes per image
    const size_t HW = (size_t)p.H * p.W, plane = (size_t)p.C * HW;
    float* wk_ws = static_cast<float*>(ws);
    const float* wk_all = RAW ? p.guidance : wk_ws;
    float* tmp_all = RAW ? wk_ws : wk_ws + (size_t)p.B * NPL * HW;
    const bool vec = p.W % 4 == 0 && aligned16(p.blur) && aligned16(p.out) && aligned16(ws) && (!RAW || aligned16(p.guidance));
    const bool keep = !PADDLE && p.keep;                 // d0' planes after the ping-pong buffer
    float* d0_all = tmp_all + (size_t)p.B * plane;
    const int G = group_size(p.B);
    for (int b0 = 0; b0 < p.B; b0 += G) {
        const int nimg = p.B - b0 < G ? p.B - b0 : G;
        const float* wk = wk_all + (size_t)b0 * NPL * HW;
        const float* blur = p.blur + (size_t)b0 * plane;
        float* out = p.out + (size_t)b0 * plane;
        float* tmp = tmp_all + (size_t)b0 * plane;
        float* d0 = keep ? d0_all + (size_t)b0 * plane : nullptr;
        if constexpr (!RAW) {
            if (keep)
                launch_prep_keep(2 * R + 1, p.guidance + (size_t)b0 * p.gch * HW, p.sparse + (size_t)b0 * HW, blur,
                                 wk_ws + (size_t)b0 * NPL * HW, d0, nimg, p.C, p.H, p.W, p.gch, p.norm_abs, stream);
            else
                launch_prep<R, PADDLE>(p.guidance + (size_t)b0 * p.gch * HW, p.sparse ? p.sparse + (size_t)b0 * HW : nullptr,
                                       wk_ws + (size_t)b0 * NPL * HW, nimg, p.H, p.W, p.gch, p.norm_abs, stream);
            ++*launches;
        }
        const Fan gfan = fan ? offset_fan(*fan, (size_t)b0 * plane) : Fan{};
        const float* cur = blur;
        float* dst = (p.iters & 1) ? out : tmp;   // ping-pong so that the last step writes out
        for (int it = 0; it < p.iters; ++it) {
            launch_step<R, PADDLE, RAW>(vec, wk, keep ? d0 : blur, cur, dst, nimg * p.C, p.C, p.H, p.W, stream,
                                        fan && it == p.iters - 1 ? &gfan : nullptr);
            ++*launches;
            cur = dst;
            dst = (dst == out) ? tmp : out;
        }
    }
    CSPN_CUDA_TRY(cudaGetLastError());
    return CSPN_OK;
}

// RAW: the caller's gates are the weight planes; the workspace holds d_1..d_{N-1} and lambda_1..lambda_{N-1} only.  The
// last adjoint step writes lambda_0 straight into grad_blur (skipped when that is null), and without grad_guidance the
// forward steps and the gather, which only feed the gate gradient, are skipped.
template <int R, bool PADDLE, bool RAW = false>
int backward_k(const Problem2D& p, const float* grad_out, float* grad_guidance, float* grad_blur, void* ws,
               cudaStream_t stream, int* launches, float* grad_sparse) {
    constexpr int NPL = RAW ? Taps<R>::NT : Taps<R>::NP;   // weight planes per image
    const size_t HW = (size_t)p.H * p.W, plane = (size_t)p.C * HW;
    const long long n = (long long)p.B * plane;
    float* wk_ws = static_cast<float*>(ws);
    const float* wk_all = RAW ? p.guidance : wk_ws;
    float* steps = RAW ? wk_ws : wk_ws + (size_t)p.B * NPL * HW;        // steps[t] = d_{t+1}, t < N-1
    // lam[t] = lambda_t; RAW keeps 1 <= t < N only, right after the steps
    float* lam = RAW ? steps + (size_t)(p.iters >= 2 ? p.iters - 2 : 0) * n : steps + (size_t)p.iters * n;
    const bool gates_grad = !RAW || grad_guidance;   // the steps and the gather feed the guidance gradient
    const bool vec = p.W % 4 == 0 && aligned16(p.blur) && aligned16(ws) && (!RAW || aligned16(p.guidance));
    const bool keep = !PADDLE && p.keep;             // d0' planes after the lambdas
    float* d0_all = lam + (size_t)p.iters * n;
    const int G = group_size(p.B);
    for (int b0 = 0; b0 < p.B; b0 += G) {
        const int nimg = p.B - b0 < G ? p.B - b0 : G;
        const size_t off = (size_t)b0 * plane;
        const float* wk = wk_all + (size_t)b0 * NPL * HW;
        const float* blur = p.blur + off;
        const float* guidance = p.guidance + (size_t)b0 * p.gch * HW;
        const float* sparse = p.sparse ? p.sparse + (size_t)b0 * HW : nullptr;
        float* d0 = keep ? d0_all + off : nullptr;
        if constexpr (!RAW) {
            if (keep)
                launch_prep_keep(2 * R + 1, guidance, sparse, blur, wk_ws + (size_t)b0 * NPL * HW, d0, nimg, p.C, p.H, p.W, p.gch,
                                 p.norm_abs, stream);
            else
                launch_prep<R, PADDLE>(guidance, sparse, wk_ws + (size_t)b0 * NPL * HW, nimg, p.H, p.W, p.gch, p.norm_abs, stream);
            ++*launches;
        }
        for (int t = 0; gates_grad && t + 1 < p.iters; ++t) {   // d_{t+1} = step(d_t)
            launch_step<R, PADDLE, RAW>(vec, wk, keep ? d0 : blur, t == 0 ? blur : steps + (size_t)(t - 1) * n + off,
                                        steps + (size_t)t * n + off, nimg * p.C, p.C, p.H, p.W, stream);
            ++*launches;
        }
        const dim3 grid((p.W + kSclTW - 1) / kSclTW, (p.H + kSclTH - 1) / kSclTH, nimg * p.C);
        for (int t = p.iters - 1; t >= 0; --t) {        // lambda_t from lambda_{t+1}
            const float* lin = (t == p.iters - 1 ? grad_out : lam + (size_t)(t + 1) * n) + off;
            float* lout = lam + (size_t)t * n + off;
            if (RAW && t == 0) {                        // lambda_0 is grad_blur
                if (!grad_blur) continue;
                lout = grad_blur + off;
            }
            adjk_kernel<R, RAW><<<grid, dim3(kSclTW, kSclTH), 0, stream>>>(wk, lin, lout, p.C, p.H, p.W);
            ++*launches;
        }
        if (!gates_grad) continue;
        float* gg = grad_guidance ? grad_guidance + (size_t)b0 * p.gch * HW : nullptr;
        if constexpr (!PADDLE) {
            if (keep) {
                gatherk_keep_kernel<R><<<dim3(grid.x, grid.y, nimg), dim3(kSclTW, kSclTH), 0, stream>>>(
                    guidance, blur, sparse, wk, steps + off, lam + off, grad_out + off, gg, grad_blur ? grad_blur + off : nullptr,
                    grad_sparse ? grad_sparse + (size_t)b0 * HW : nullptr, n, p.iters, p.C, p.H, p.W, p.gch, p.norm_abs);
                ++*launches;
                continue;
            }
        }
        gatherk_kernel<R, PADDLE, RAW><<<dim3(grid.x, grid.y, nimg), dim3(kSclTW, kSclTH), 0, stream>>>(
                guidance, blur, sparse, wk, steps + off, lam + off, grad_out + off, gg, grad_blur && !RAW ? grad_blur + off : nullptr,
                n, p.iters, p.C, p.H, p.W, p.gch, p.norm_abs);
        ++*launches;
    }
    CSPN_CUDA_TRY(cudaGetLastError());
    return CSPN_OK;
}

// Aggregation (DESIGN.md section 4.20), the normalised family: out = sum_j sw_j * d_{s_j}, steps s_0 < ... < s_{nw-1} = N.
// Workspace: the K*K weight planes, two ping-pong planes (out is the running sum, so no iterate is stored there), keep's d0'.
template <int R>
int aggregate_forward_k(const Problem2D& p, const float* sw, const int* steps, int nw, void* ws, cudaStream_t stream,
                        int* launches) {
    constexpr int NPL = Taps<R>::NP;
    const size_t HW = (size_t)p.H * p.W, plane = (size_t)p.C * HW;
    float* wk_ws = static_cast<float*>(ws);
    float* buf[2] = {wk_ws + (size_t)p.B * NPL * HW, wk_ws + (size_t)p.B * NPL * HW + (size_t)p.B * plane};
    float* d0_all = buf[1] + (size_t)p.B * plane;
    const bool vec = p.W % 4 == 0 && aligned16(p.blur) && aligned16(p.out) && aligned16(ws) && aligned16(sw);
    const dim3 vgrid((p.W + kVecTW - 1) / kVecTW, (p.H + kVecTH - 1) / kVecTH), sgrid((p.W + kSclTW - 1) / kSclTW, (p.H + kSclTH - 1) / kSclTH);
    const int G = group_size(p.B);
    for (int b0 = 0; b0 < p.B; b0 += G) {
        const int nimg = p.B - b0 < G ? p.B - b0 : G;
        const size_t off = (size_t)b0 * plane;
        const float* wk = wk_ws + (size_t)b0 * NPL * HW;
        const float* blur = p.blur + off;
        float* d0 = p.keep ? d0_all + off : nullptr;
        if (p.keep)
            launch_prep_keep(2 * R + 1, p.guidance + (size_t)b0 * p.gch * HW, p.sparse + (size_t)b0 * HW, blur, wk_ws + (size_t)b0 * NPL * HW,
                             d0, nimg, p.C, p.H, p.W, p.gch, p.norm_abs, stream);
        else
            launch_prep<R, false>(p.guidance + (size_t)b0 * p.gch * HW, p.sparse ? p.sparse + (size_t)b0 * HW : nullptr,
                                  wk_ws + (size_t)b0 * NPL * HW, nimg, p.H, p.W, p.gch, p.norm_abs, stream);
        ++*launches;
        const float* cur = blur;
        for (int t = 0, j = 0; t < p.iters; ++t) {           // d_{t+1} = step(d_t)
            float* dst = t + 1 == p.iters ? nullptr : buf[t & 1] + off;
            if (steps[j] == t + 1) {
                const float* lam = sw + ((size_t)b0 * nw + j) * HW;
                const int nbc = nimg * p.C;
                if (vec)
                    stepk_agg_vec_kernel<R><<<dim3(vgrid.x, vgrid.y, nbc), dim3(16, 16), 0, stream>>>(
                            wk, p.keep ? d0 : blur, cur, dst, lam, nw, p.out + off, j == 0, p.C, p.H, p.W);
                else
                    stepk_agg_scalar_kernel<R><<<dim3(sgrid.x, sgrid.y, nbc), dim3(kSclTW, kSclTH), 0, stream>>>(
                            wk, p.keep ? d0 : blur, cur, dst, lam, nw, p.out + off, j == 0, p.C, p.H, p.W);
                ++j;
            } else {
                launch_step<R, false>(vec, wk, p.keep ? d0 : blur, cur, dst, nimg * p.C, p.C, p.H, p.W, stream);
            }
            ++*launches;
            cur = dst;
        }
    }
    CSPN_CUDA_TRY(cudaGetLastError());
    return CSPN_OK;
}

// Backward: prep, N forward steps that keep d_1..d_N, the step-weight gradient with mu_N = sw_{nw-1} * grad_out, N adjoint
// steps mu_t = adj(mu_{t+1}) (+ sw_j * grad_out where t = s_j), and the gather of backward_k reading mu_N as its last adjoint.
// Workspace: the weight planes, d_1..d_N, mu_0..mu_N, keep's d0'.
template <int R>
int aggregate_backward_k(const Problem2D& p, const float* sw, const int* steps, int nw, const float* grad_out, float* grad_guidance,
                         float* grad_blur, float* grad_sparse, float* grad_sw, void* ws, cudaStream_t stream, int* launches) {
    constexpr int NPL = Taps<R>::NP;
    const int N = p.iters;
    const size_t HW = (size_t)p.H * p.W, plane = (size_t)p.C * HW;
    const long long n = (long long)p.B * plane;
    float* wk_ws = static_cast<float*>(ws);
    float* its = wk_ws + (size_t)p.B * NPL * HW;          // its[t] = d_{t+1}, t < N
    float* lam = its + (size_t)N * n;                     // lam[t] = mu_t, t <= N
    float* d0_all = lam + (size_t)(N + 1) * n;
    const bool vec = p.W % 4 == 0 && aligned16(p.blur) && aligned16(ws);
    const int G = group_size(p.B);
    for (int b0 = 0; b0 < p.B; b0 += G) {
        const int nimg = p.B - b0 < G ? p.B - b0 : G;
        const size_t off = (size_t)b0 * plane;
        const float* wk = wk_ws + (size_t)b0 * NPL * HW;
        const float* blur = p.blur + off;
        const float* guidance = p.guidance + (size_t)b0 * p.gch * HW;
        const float* sparse = p.sparse ? p.sparse + (size_t)b0 * HW : nullptr;
        const float* swg = sw + (size_t)b0 * nw * HW;
        float* d0 = p.keep ? d0_all + off : nullptr;
        if (p.keep)
            launch_prep_keep(2 * R + 1, guidance, sparse, blur, wk_ws + (size_t)b0 * NPL * HW, d0, nimg, p.C, p.H, p.W, p.gch,
                             p.norm_abs, stream);
        else
            launch_prep<R, false>(guidance, sparse, wk_ws + (size_t)b0 * NPL * HW, nimg, p.H, p.W, p.gch, p.norm_abs, stream);
        ++*launches;
        for (int t = 0; t < N; ++t) {
            launch_step<R, false>(vec, wk, p.keep ? d0 : blur, t == 0 ? blur : its + (size_t)(t - 1) * n + off,
                                  its + (size_t)t * n + off, nimg * p.C, p.C, p.H, p.W, stream);
            ++*launches;
        }
        float* mu_n = lam + (size_t)N * n + off;
        for (int j0 = 0; j0 < nw; j0 += kAggStepsPerLaunch) {
            StepSel sel{};
            const int ns = nw - j0 < kAggStepsPerLaunch ? nw - j0 : kAggStepsPerLaunch;
            for (int j = 0; j < ns; ++j) sel.s[j] = steps[j0 + j];
            agg_gradw_kernel<<<dim3((unsigned)((HW + 255) / 256), 1, nimg), 256, 0, stream>>>(
                    grad_out + off, its + off, n, swg, grad_sw ? grad_sw + (size_t)b0 * nw * HW : nullptr,
                    j0 + ns == nw ? mu_n : nullptr, sel, j0, ns, nw, p.C, (long long)HW);
            ++*launches;
        }
        const dim3 grid((p.W + kSclTW - 1) / kSclTW, (p.H + kSclTH - 1) / kSclTH, nimg * p.C);
        for (int t = N - 1, j = nw - 2; t >= 0; --t) {    // mu_t from mu_{t+1}
            const float* lin = lam + (size_t)(t + 1) * n + off;
            float* lout = lam + (size_t)t * n + off;
            if (j >= 0 && steps[j] == t) {
                adjk_inject_kernel<R><<<grid, dim3(kSclTW, kSclTH), 0, stream>>>(wk, lin, lout, swg + (size_t)j * HW, nw,
                                                                                 grad_out + off, p.C, p.H, p.W);
                --j;
            } else {
                adjk_kernel<R, false><<<grid, dim3(kSclTW, kSclTH), 0, stream>>>(wk, lin, lout, p.C, p.H, p.W);
            }
            ++*launches;
        }
        float* gg = grad_guidance ? grad_guidance + (size_t)b0 * p.gch * HW : nullptr;
        float* gb = grad_blur ? grad_blur + off : nullptr;
        const dim3 ggrid(grid.x, grid.y, nimg);
        if (p.keep)
            gatherk_keep_kernel<R><<<ggrid, dim3(kSclTW, kSclTH), 0, stream>>>(
                    guidance, blur, sparse, wk, its + off, lam + off, mu_n, gg, gb, grad_sparse ? grad_sparse + (size_t)b0 * HW : nullptr,
                    n, N, p.C, p.H, p.W, p.gch, p.norm_abs);
        else
            gatherk_kernel<R, false, false><<<ggrid, dim3(kSclTW, kSclTH), 0, stream>>>(
                    guidance, blur, sparse, wk, its + off, lam + off, mu_n, gg, gb, n, N, p.C, p.H, p.W, p.gch, p.norm_abs);
        ++*launches;
    }
    CSPN_CUDA_TRY(cudaGetLastError());
    return CSPN_OK;
}

// What the three families' fronts do differently; their kernels differ by the PADDLE / RAW flags (see with_kernels)
struct FamilyTraits {
    const char* name;        // follows "KxK 2D" in messages
    bool zero_grad_first;    // grad_guidance is zero-filled before every run, not only at iters == 0: channels >= K*K-1 and
                             // taps that read the padding get no store.  The other two families write every guidance
                             // gradient (each g_j(p) feeds pixel p alone; a tap that reads the padding gets 0)
    bool checks_grid_y;
    bool no_grad_is_no_op;   // a backward that is asked for neither gradient launches nothing
};

const FamilyTraits& traits(Family family) {
    static const FamilyTraits t[] = {{"", true, false, false}, {" 'paddle'", false, false, false}, {" gates", false, true, true}};
    return t[(int)family];
}

// f(R, PADDLE, RAW) as integral constants for the K x K kernels of `family`.  The normalised family's K = 3 is the 3x3
// operator, whose backward falls back to these kernels (cspn2d_bwd.cu); its forward is never sent here.
template <class F>
int with_kernels(int K, Family family, F&& f) {
    using std::integral_constant;
    constexpr std::true_type yes{};
    constexpr std::false_type no{};
    const auto radius = [&](auto paddle, auto raw) {
        return K == 3 ? f(integral_constant<int, 1>{}, paddle, raw)
             : K == 5 ? f(integral_constant<int, 2>{}, paddle, raw) : f(integral_constant<int, 3>{}, paddle, raw);
    };
    return family == Family::Normalised ? radius(no, no) : family == Family::Paddle ? radius(yes, no) : radius(yes, yes);
}

// The workspace holds what `need` says, and the launch grids (z = image*channel, y = rows of 8) take the problem
int check_launch(const Problem2D& p, int K, const FamilyTraits& t, const char* what, size_t need, const void* ws, size_t ws_bytes) {
    if (need && (!ws || ws_bytes < need)) {
        set_error("%dx%d 2D%s %s needs %zu workspace bytes, got %zu", K, K, t.name, what, need, ws ? ws_bytes : (size_t)0);
        return CSPN_ERR_WORKSPACE;
    }
    if ((long long)p.B * p.C > 65535) {
        set_error("%dx%d 2D%s %s: B*C=%lld exceeds gridDim.z", K, K, t.name, what, (long long)p.B * p.C);
        return CSPN_ERR_UNSUPPORTED;
    }
    if (t.checks_grid_y && (p.H + kSclTH - 1) / kSclTH > 65535) {
        set_error("%dx%d 2D%s %s: H=%d exceeds gridDim.y", K, K, t.name, what, p.H);
        return CSPN_ERR_UNSUPPORTED;
    }
    return CSPN_OK;
}

}  // namespace

// Normalised and 'paddle': K*K weight planes per image and the ping-pong buffer.  Gates: the caller's gates are the weight
// planes, and a single step writes `out` directly.
// keep (Normalised): the d0' planes of the keep-sparse mode follow
void launch_prep_keep(int K, const float* guidance, const float* sparse, const float* blur, float* wk, float* d0, int B, int C,
                      int H, int W, int gch, int norm_abs, cudaStream_t stream) {
    const dim3 grid((W + 31) / 32, (H + 7) / 8, B), block(32, 8);
    if (K == 3) prepk_keep_kernel<1><<<grid, block, 0, stream>>>(guidance, sparse, blur, wk, d0, C, H, W, gch, norm_abs);
    else if (K == 5) prepk_keep_kernel<2><<<grid, block, 0, stream>>>(guidance, sparse, blur, wk, d0, C, H, W, gch, norm_abs);
    else prepk_keep_kernel<3><<<grid, block, 0, stream>>>(guidance, sparse, blur, wk, d0, C, H, W, gch, norm_abs);
}

size_t widek_workspace_bytes(int B, int C, int H, int W, int K, int iters, Family family, bool keep) {
    if (iters <= 0) return 0;
    const size_t HW = (size_t)H * W;
    if (family == Family::Gates) return iters >= 2 ? sizeof(float) * (size_t)B * C * HW : 0;
    return sizeof(float) * ((size_t)B * K * K * HW + (keep ? 2 : 1) * (size_t)B * C * HW);
}

// The weight planes as above, then d_1..d_{N-1} and the lambdas: 2N planes of B*C images, 2N-2 for gates (see backward_k)
size_t widek_bwd_workspace_bytes(int B, int C, int H, int W, int K, int iters, Family family, bool keep) {
    if (iters <= 0) return 0;
    const size_t HW = (size_t)H * W;
    if (family == Family::Gates) return sizeof(float) * (2 * (size_t)iters - 2) * B * C * HW;
    return sizeof(float) * ((size_t)B * K * K * HW + (2 * (size_t)iters + (keep ? 1 : 0)) * B * C * HW);
}

int widek_forward(const Problem2D& p, int K, Family family, void* ws, size_t ws_bytes, cudaStream_t stream, int* launches,
                  const Fan* fan) {
    if (p.iters == 0) {
        CSPN_CUDA_TRY(cudaMemcpyAsync(p.out, p.blur, (size_t)p.B * p.C * p.H * p.W * sizeof(float), cudaMemcpyDeviceToDevice, stream));
        return CSPN_OK;
    }
    const int rc = check_launch(p, K, traits(family), "path", widek_workspace_bytes(p.B, p.C, p.H, p.W, K, p.iters, family, p.keep),
                                ws, ws_bytes);
    if (rc != CSPN_OK) return rc;
    return with_kernels(K, family, [&](auto R, auto PADDLE, auto RAW) {
        return forward_k<R(), PADDLE(), RAW()>(p, ws, stream, launches, fan);
    });
}

int widek_backward(const Problem2D& p, int K, Family family, const float* grad_out, float* grad_guidance, float* grad_blur,
                   void* ws, size_t ws_bytes, cudaStream_t stream, int* launches, float* grad_sparse) {
    const FamilyTraits& t = traits(family);
    const size_t HW = (size_t)p.H * p.W, n = (size_t)p.B * p.C * HW;
    if (grad_guidance && (t.zero_grad_first || p.iters == 0))
        CSPN_CUDA_TRY(cudaMemsetAsync(grad_guidance, 0, (size_t)p.B * p.gch * HW * sizeof(float), stream));
    if (p.iters == 0) {   // the identity: no dependence on the guidance
        if (grad_blur) CSPN_CUDA_TRY(cudaMemcpyAsync(grad_blur, grad_out, n * sizeof(float), cudaMemcpyDeviceToDevice, stream));
        return CSPN_OK;
    }
    const int rc = check_launch(p, K, t, "backward", widek_bwd_workspace_bytes(p.B, p.C, p.H, p.W, K, p.iters, family, p.keep), ws,
                                ws_bytes);
    if (rc != CSPN_OK) return rc;
    if (t.no_grad_is_no_op && !grad_guidance && !grad_blur) return CSPN_OK;
    return with_kernels(K, family, [&](auto R, auto PADDLE, auto RAW) {
        return backward_k<R(), PADDLE(), RAW()>(p, grad_out, grad_guidance, grad_blur, ws, stream, launches, grad_sparse);
    });
}

size_t aggregate2d_workspace_bytes(int B, int C, int H, int W, int K, bool keep) {
    const size_t HW = (size_t)H * W;
    return sizeof(float) * ((size_t)B * K * K * HW + (keep ? 3 : 2) * (size_t)B * C * HW);
}

size_t aggregate2d_bwd_workspace_bytes(int B, int C, int H, int W, int K, int N, bool keep) {
    const size_t HW = (size_t)H * W;
    return sizeof(float) * ((size_t)B * K * K * HW + (2 * (size_t)N + 1 + (keep ? 1 : 0)) * B * C * HW);
}

int aggregate2d_forward(const Problem2D& p, int K, const float* step_weight, const int* steps, int n_steps, void* ws,
                        size_t ws_bytes, cudaStream_t stream, int* launches) {
    const int rc = check_launch(p, K, traits(Family::Normalised), "aggregation",
                                aggregate2d_workspace_bytes(p.B, p.C, p.H, p.W, K, p.keep), ws, ws_bytes);
    if (rc != CSPN_OK) return rc;
    return with_kernels(K, Family::Normalised, [&](auto R, auto, auto) {
        return aggregate_forward_k<R()>(p, step_weight, steps, n_steps, ws, stream, launches);
    });
}

int aggregate2d_backward(const Problem2D& p, int K, const float* step_weight, const int* steps, int n_steps, const float* grad_out,
                         float* grad_guidance, float* grad_blur, float* grad_sparse, float* grad_step_weight, void* ws,
                         size_t ws_bytes, cudaStream_t stream, int* launches) {
    const int rc = check_launch(p, K, traits(Family::Normalised), "aggregation backward",
                                aggregate2d_bwd_workspace_bytes(p.B, p.C, p.H, p.W, K, p.iters, p.keep), ws, ws_bytes);
    if (rc != CSPN_OK) return rc;
    if (grad_guidance)   // channels >= K*K-1 and taps that read the padding get no store, as in widek_backward
        CSPN_CUDA_TRY(cudaMemsetAsync(grad_guidance, 0, (size_t)p.B * p.gch * p.H * p.W * sizeof(float), stream));
    return with_kernels(K, Family::Normalised, [&](auto R, auto, auto) {
        return aggregate_backward_k<R()>(p, step_weight, steps, n_steps, grad_out, grad_guidance, grad_blur, grad_sparse,
                                         grad_step_weight, ws, stream, launches);
    });
}

}  // namespace cspn
