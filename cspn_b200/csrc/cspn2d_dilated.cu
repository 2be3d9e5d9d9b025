// Dilated K x K propagation with a centre weight on the initial depth and a learned confidence for the samples: PENet's
// DA-CSPN++ (Hu et al., ICRA 2021) step (DESIGN.md section 4.22).  kernel (B, K*K, H, W) holds the weights as given, shared
// by the C channels; channel j = i*K + l weights the value at p + dil*(i - R, l - R), R = (K - 1) / 2 (F.unfold's row
// order), and the centre channel c = (K*K - 1) / 2 weights d_0(p).  blur (B, C, H, W) is d_0; sparse s and confidence m are
// (B, 1, H, W), both or neither.  A read outside the image is 0.
//
//   u_t(p)     = fma over j = K*K-1 down to 0, j != c, of w_j(p) * d_t(p + dil*o_j), starting from w_c(p) * d_0(p)
//   d_{t+1}(p) = m*s + (1 - m)*u_t(p)       (with samples; d_{t+1} = u_t without), out = d_N
//
// Every product outside the FMA chain and every sum is rounded on its own.  The j order is the K x K kernels' tap order
// (their tap k reads offset (R - t, R - l), which is unfold row K*K-1 - (t*K + l)), so at dil = 1 with w_c = 0 and no samples
// a step gives affinity_propagate's bits.  The confidence is not folded into the weights: with an infinite m the folded sum
// (1 - m) w_j d + m s can meet inf - inf where (1 - m) u does not, and the NaN masks would differ from the composition's.
//
// Backward, lambda_N = grad_out, a = 1 - m (a = 1 without samples), mu_t = a * lambda_{t+1}:
//   lambda_t(q)      = fma over j = K*K-1 down to 0, j != c, source q - dil*o_j inside the image, of w_j * mu_t there
//   grad_blur        = lambda_0 + sum_t w_c mu_t                                     (fma, t ascending)
//   grad_kernel_j(p) = sum_t sum_c mu_t d_t(p + dil*o_j),  grad_kernel_c = sum_t sum_c mu_t d_0    (fma, t then c ascending;
//                      a tap outside the image adds mu * 0)
//   grad_conf(p)     = sum_t ((sum_c lambda_{t+1}) s - sum_c lambda_{t+1} u_t),  grad_sparse(p) = sum_t m sum_c lambda_{t+1}
//                      (t then c ascending; the lambda sum by adds, the lambda u sum by fma)
// with u_t recomputed in the forward's order.  Only a kernel or confidence gradient needs d_1 .. d_{N-1}.
//
// Kernels (sm_90a):
//   step      one launch per step, grid z = image * channel; a tile of d_t with a dil*R halo staged in shared memory (zeros
//             outside the image); 4 pixels per thread with LDG.128 weights when W % 4 == 0 and the planes are 16-byte
//             aligned, else 1; both give the same bits;
//   adjoint   one launch per step, the transposed stencil over a staged tile of mu_t, one pixel per thread;
//   finalize  one launch: a thread per pixel and kernel row for grad_kernel, and a thread per pixel for the others,
//             each over all channels and steps.
// No atomics and no memsets (except the N = 0 backward's zero gradients); every output word is written by one thread.
#include "cspn2d_stencil.cuh"

namespace cspn {
namespace {

constexpr int kTX = 32, kTY = 8, kRows = 2;          // threads per CTA (x, y); each thread runs kRows tile rows
constexpr int kTH = kTY * kRows;                     // tile height
constexpr int kFinThreads = 128;

template <int K, int VEC, bool SAMP>
__global__ void __launch_bounds__(kTX * kTY)
dil_step_kernel(const float* __restrict__ kern, const float* __restrict__ d0, const float* __restrict__ cur,
                const float* __restrict__ sparse, const float* __restrict__ conf, float* __restrict__ dst, int C, int H, int W,
                int dil) {
    constexpr int R = (K - 1) / 2, KK = K * K, CEN = KK / 2;
    extern __shared__ float tile[];
    const int TW = kTX * VEC, h = dil * R, pitch = TW + 2 * h;
    const int x0 = blockIdx.x * TW, y0 = blockIdx.y * kTH, bc = blockIdx.z, b = bc / C;
    const size_t HW = (size_t)H * W;
    stage<kTX, kTY, kTH>(tile, pitch, cur + (size_t)bc * HW, nullptr, x0, y0, h, H, W);
    __syncthreads();
    const float* wk = kern + (size_t)b * KK * HW;
    const int tx = threadIdx.x * VEC, x = x0 + tx;
    if (x >= W) return;
#pragma unroll 1
    for (int r = 0; r < kRows; ++r) {
        const int ty = threadIdx.y + r * kTY, y = y0 + ty;
        if (y >= H) return;
        const size_t p = (size_t)y * W + x, o = (size_t)bc * HW + p;
        const float* t0 = tile + (ty + h) * pitch + tx + h;
        if constexpr (VEC == 4) {
            const float4 wc = ld4(wk + CEN * HW + p), dd = ld4(d0 + o);
            float u0 = __fmul_rn(wc.x, dd.x), u1 = __fmul_rn(wc.y, dd.y), u2 = __fmul_rn(wc.z, dd.z), u3 = __fmul_rn(wc.w, dd.w);
#pragma unroll
            for (int j = KK - 1; j >= 0; --j) {
                if (j == CEN) continue;
                const float4 w = ld4(wk + j * HW + p);
                const float* s = t0 + dil * ((j / K - R) * pitch + (j % K - R));
                u0 = fmaf(w.x, s[0], u0);
                u1 = fmaf(w.y, s[1], u1);
                u2 = fmaf(w.z, s[2], u2);
                u3 = fmaf(w.w, s[3], u3);
            }
            if constexpr (SAMP) {
                const float4 m = ld4(conf + (size_t)b * HW + p), sv = ld4(sparse + (size_t)b * HW + p);
                u0 = blend(m.x, sv.x, u0);
                u1 = blend(m.y, sv.y, u1);
                u2 = blend(m.z, sv.z, u2);
                u3 = blend(m.w, sv.w, u3);
            }
            *reinterpret_cast<float4*>(dst + o) = make_float4(u0, u1, u2, u3);
        } else {
            float u = __fmul_rn(__ldg(wk + CEN * HW + p), __ldg(d0 + o));
#pragma unroll
            for (int j = KK - 1; j >= 0; --j) {
                if (j == CEN) continue;
                u = fmaf(__ldg(wk + j * HW + p), t0[dil * ((j / K - R) * pitch + (j % K - R))], u);
            }
            if constexpr (SAMP) u = blend(__ldg(conf + (size_t)b * HW + p), __ldg(sparse + (size_t)b * HW + p), u);
            dst[o] = u;
        }
    }
}

// lambda_t(q) = sum_j w_j(q - dil*o_j) mu_t(q - dil*o_j), sources inside the image only; mu_t = (1 - m) lambda_{t+1}
// (conf) or lambda_{t+1}
template <int K>
__global__ void __launch_bounds__(kTX * kTY)
dil_adjoint_kernel(const float* __restrict__ kern, const float* __restrict__ lam_in, const float* __restrict__ conf,
                   float* __restrict__ lam_out, int C, int H, int W, int dil) {
    constexpr int R = (K - 1) / 2, KK = K * K, CEN = KK / 2;
    extern __shared__ float tile[];
    const int h = dil * R, pitch = kTX + 2 * h;
    const int x0 = blockIdx.x * kTX, y0 = blockIdx.y * kTH, bc = blockIdx.z, b = bc / C;
    const size_t HW = (size_t)H * W;
    stage<kTX, kTY, kTH>(tile, pitch, lam_in + (size_t)bc * HW, conf ? conf + (size_t)b * HW : nullptr, x0, y0, h, H, W);
    __syncthreads();
    const float* wk = kern + (size_t)b * KK * HW;
    const int tx = threadIdx.x, x = x0 + tx;
    if (x >= W) return;
#pragma unroll 1
    for (int r = 0; r < kRows; ++r) {
        const int ty = threadIdx.y + r * kTY, y = y0 + ty;
        if (y >= H) return;
        const float* t0 = tile + (ty + h) * pitch + tx + h;
        float acc = 0.f;
#pragma unroll 1
        for (int i = K - 1; i >= 0; --i) {                            // j = i*K + l descending
            const int oy = dil * (i - R), ys = y - oy;
#pragma unroll
            for (int l = K - 1; l >= 0; --l) {
                if (i * K + l == CEN) continue;
                const int ox = dil * (l - R), xs = x - ox;
                if (in_image(ys, xs, H, W)) acc = fmaf(__ldg(wk + (i * K + l) * HW + (size_t)ys * W + xs), t0[-oy * pitch - ox], acc);
            }
        }
        lam_out[(size_t)bc * HW + (size_t)y * W + x] = acc;
    }
}

// The gradients of pixel p of image b.  lams holds lambda_0 .. lambda_{N-1} (lambda_N is grad_out), iters d_1 .. d_{N-1}
// (d_0 is blur), each P = B*C*H*W floats.  ITER (a kernel or confidence gradient): grid z = K + 1, slice i < K forms
// grad_kernel of the taps in kernel row i, slice K the per-pixel rest; without ITER grid z = 1 and no iterate is read.
// Splitting the rows keeps the K = 7 accumulators in registers.
template <int K, bool SAMP, bool ITER>
__global__ void __launch_bounds__(kFinThreads)
dil_finalize_kernel(const float* __restrict__ kern, const float* __restrict__ d0, const float* __restrict__ sparse,
                    const float* __restrict__ conf, const float* __restrict__ grad_out, const float* __restrict__ iters,
                    const float* __restrict__ lams, float* __restrict__ grad_kern, float* __restrict__ grad_blur,
                    float* __restrict__ grad_sparse, float* __restrict__ grad_conf, int N, size_t P, int C, int H, int W, int dil) {
    constexpr int R = (K - 1) / 2, KK = K * K, CEN = KK / 2;
    const size_t HW = (size_t)H * W;
    const long long pl = (long long)blockIdx.x * kFinThreads + threadIdx.x;
    if (pl >= (long long)HW) return;
    const size_t p = (size_t)pl;
    const int b = blockIdx.y, y = (int)(p / W), x = (int)(p % W);
    const float* wk = kern + (size_t)b * KK * HW + p;
    const float m = SAMP ? __ldg(conf + (size_t)b * HW + p) : 0.f;
    const float a = SAMP ? __fsub_rn(1.f, m) : 1.f;
    auto lam = [&](int t, size_t o) { return t == N ? __ldg(grad_out + o) : __ldg(lams + (size_t)t * P + o); };
    auto iterate = [&](int t, size_t plane) { return t == 0 ? d0 + plane : iters + (size_t)(t - 1) * P + plane; };
    if (ITER && (int)blockIdx.z < K) {
        if (!grad_kern) return;
        const int i = blockIdx.z, ys = y + dil * (i - R);
        float gw[K];
#pragma unroll
        for (int l = 0; l < K; ++l) gw[l] = 0.f;
        for (int t = 0; t < N; ++t)
            for (int c = 0; c < C; ++c) {
                const size_t plane = ((size_t)b * C + c) * HW;
                const float l0 = lam(t + 1, plane + p), mu = SAMP ? __fmul_rn(a, l0) : l0;
                const float* dt = iterate(t, plane);
#pragma unroll
                for (int l = 0; l < K; ++l) {
                    const int xs = x + dil * (l - R);
                    float v;
                    if (i * K + l == CEN) v = __ldg(d0 + plane + p);
                    else v = in_image(ys, xs, H, W) ? __ldg(dt + (size_t)ys * W + xs) : 0.f;
                    gw[l] = fmaf(mu, v, gw[l]);
                }
            }
#pragma unroll
        for (int l = 0; l < K; ++l) grad_kern[((size_t)b * KK + i * K + l) * HW + p] = gw[l];
        return;
    }
    const float wc = __ldg(wk + CEN * HW);
    if (grad_blur) {
        for (int c = 0; c < C; ++c) {
            const size_t o = ((size_t)b * C + c) * HW + p;
            float g = __ldg(lams + o);
            for (int t = 0; t < N; ++t) g = fmaf(wc, SAMP ? __fmul_rn(a, lam(t + 1, o)) : lam(t + 1, o), g);
            grad_blur[o] = g;
        }
    }
    if constexpr (SAMP) {
        if (!grad_sparse && !grad_conf) return;
        const float s = __ldg(sparse + (size_t)b * HW + p);
        float gm = 0.f, gs = 0.f;
        for (int t = 0; t < N; ++t) {
            float A = 0.f, Bs = 0.f;
            for (int c = 0; c < C; ++c) {
                const size_t plane = ((size_t)b * C + c) * HW;
                const float l0 = lam(t + 1, plane + p);
                A = __fadd_rn(A, l0);
                if (ITER && grad_conf) {
                    const float* dt = iterate(t, plane);
                    float u = __fmul_rn(wc, __ldg(d0 + plane + p));
#pragma unroll 1
                    for (int i = K - 1; i >= 0; --i) {                // j = i*K + l descending, the forward's order
                        const int ys = y + dil * (i - R);
#pragma unroll
                        for (int l = K - 1; l >= 0; --l) {
                            if (i * K + l == CEN) continue;
                            const int xs = x + dil * (l - R);
                            u = fmaf(__ldg(wk + (i * K + l) * HW), in_image(ys, xs, H, W) ? __ldg(dt + (size_t)ys * W + xs) : 0.f, u);
                        }
                    }
                    Bs = fmaf(l0, u, Bs);
                }
            }
            gm = __fadd_rn(gm, __fsub_rn(__fmul_rn(A, s), Bs));
            gs = __fadd_rn(gs, __fmul_rn(m, A));
        }
        if (ITER && grad_conf) grad_conf[(size_t)b * HW + p] = gm;
        if (grad_sparse) grad_sparse[(size_t)b * HW + p] = gs;
    }
}

size_t tile_smem(int VEC, int h) { return (size_t)(kTH + 2 * h) * (kTX * VEC + 2 * h) * sizeof(float); }

template <int K>
int launch_step(bool vec, const float* kern, const float* d0, const float* cur, const float* sparse, const float* conf, float* dst,
                int B, int C, int H, int W, int dil, cudaStream_t st) {
    const int h = dil * (K - 1) / 2;
    const int VEC = vec ? 4 : 1;
    const dim3 grid((unsigned)ceil_div(W, kTX * VEC), (unsigned)ceil_div(H, kTH), (unsigned)(B * C)), block(kTX, kTY);
    const size_t sm = tile_smem(VEC, h);
    if (vec && sparse)
        dil_step_kernel<K, 4, true><<<grid, block, sm, st>>>(kern, d0, cur, sparse, conf, dst, C, H, W, dil);
    else if (vec)
        dil_step_kernel<K, 4, false><<<grid, block, sm, st>>>(kern, d0, cur, sparse, conf, dst, C, H, W, dil);
    else if (sparse)
        dil_step_kernel<K, 1, true><<<grid, block, sm, st>>>(kern, d0, cur, sparse, conf, dst, C, H, W, dil);
    else
        dil_step_kernel<K, 1, false><<<grid, block, sm, st>>>(kern, d0, cur, sparse, conf, dst, C, H, W, dil);
    CSPN_CUDA_TRY(cudaGetLastError());
    return CSPN_OK;
}

template <int K>
int forward_k(const float* kern, const float* blur, const float* sparse, const float* conf, float* out, int B, int C, int H, int W,
              int dil, int N, void* ws, cudaStream_t st, int* launches) {
    float* buf = static_cast<float*>(ws);
    const bool vec = vec_ok(W, {kern, blur, sparse, conf, out, N > 1 ? buf : nullptr});
    const float* cur = blur;
    for (int t = 0; t < N; ++t) {
        float* dst = ((N - 1 - t) & 1) ? buf : out;      // d_N lands in out; the others alternate with the one buffer
        const int rc = launch_step<K>(vec, kern, blur, cur, sparse, conf, dst, B, C, H, W, dil, st);
        if (rc != CSPN_OK) return rc;
        cur = dst;
    }
    *launches = N;
    return CSPN_OK;
}

template <int K>
int backward_k(const float* kern, const float* blur, const float* sparse, const float* conf, const float* grad_out, float* grad_kern,
               float* grad_blur, float* grad_sparse, float* grad_conf, int B, int C, int H, int W, int dil, int N, void* ws,
               cudaStream_t st, int* launches) {
    const size_t P = (size_t)B * C * H * W;
    float* lams = static_cast<float*>(ws);                   // lambda_0 .. lambda_{N-1}
    float* iters = lams + (size_t)N * P;                     // d_1 .. d_{N-1}
    const bool iter = grad_kern || grad_conf;
    int nl = 0;
    if (iter) {
        const bool vec = vec_ok(W, {kern, blur, sparse, conf, N > 1 ? iters : nullptr});
        for (int t = 0; t + 1 < N; ++t) {
            const int rc = launch_step<K>(vec, kern, blur, t == 0 ? blur : iters + (size_t)(t - 1) * P, sparse, conf,
                                          iters + (size_t)t * P, B, C, H, W, dil, st);
            if (rc != CSPN_OK) return rc;
            ++nl;
        }
    }
    const int t_end = grad_blur ? 0 : 1;                      // lambda_0 feeds grad_blur only
    const int h = dil * (K - 1) / 2;
    const dim3 grid((unsigned)ceil_div(W, kTX), (unsigned)ceil_div(H, kTH), (unsigned)(B * C)), block(kTX, kTY);
    for (int t = N - 1; t >= t_end; --t) {
        dil_adjoint_kernel<K><<<grid, block, tile_smem(1, h), st>>>(kern, t + 1 == N ? grad_out : lams + (size_t)(t + 1) * P, conf,
                                                                    lams + (size_t)t * P, C, H, W, dil);
        CSPN_CUDA_TRY(cudaGetLastError());
        ++nl;
    }
    const dim3 fg((unsigned)ceil_div((long long)H * W, kFinThreads), (unsigned)B, iter ? K + 1 : 1);
#define CSPN_DIL_FIN(S, I)                                                                                                      \
    dil_finalize_kernel<K, S, I><<<fg, kFinThreads, 0, st>>>(kern, blur, sparse, conf, grad_out, iters, lams, grad_kern, grad_blur, \
                                                             grad_sparse, grad_conf, N, P, C, H, W, dil)
    if (sparse && iter) CSPN_DIL_FIN(true, true);
    else if (sparse) CSPN_DIL_FIN(true, false);
    else if (iter) CSPN_DIL_FIN(false, true);
    else CSPN_DIL_FIN(false, false);
#undef CSPN_DIL_FIN
    CSPN_CUDA_TRY(cudaGetLastError());
    *launches = nl + 1;
    return CSPN_OK;
}

}  // namespace

int dilated2d_launchable(int B, int C, int H, int W, const char** why) {
    if ((long long)B * C > 65535) { *why = "B*C exceeds gridDim.z (65535)"; return 0; }
    if (ceil_div(H, kTH) > 65535) { *why = "ceil(H/16) exceeds gridDim.y (65535)"; return 0; }
    return 1;
}

size_t dilated2d_workspace_bytes(int B, int C, int H, int W, int N) {
    return N >= 2 ? (size_t)B * C * H * W * sizeof(float) : 0;
}

size_t dilated2d_bwd_workspace_bytes(int B, int C, int H, int W, int N) {
    return N >= 1 ? (size_t)(2 * N - 1) * B * C * H * W * sizeof(float) : 0;
}

int dilated2d_forward(const float* kern, const float* blur, const float* sparse, const float* conf, float* out, int B, int C, int H,
                      int W, int K, int dil, int N, void* ws, cudaStream_t st, int* launches) {
    if (N == 0) {
        CSPN_CUDA_TRY(cudaMemcpyAsync(out, blur, (size_t)B * C * H * W * sizeof(float), cudaMemcpyDeviceToDevice, st));
        *launches = 0;
        return CSPN_OK;
    }
    switch (K) {
        case 3: return forward_k<3>(kern, blur, sparse, conf, out, B, C, H, W, dil, N, ws, st, launches);
        case 5: return forward_k<5>(kern, blur, sparse, conf, out, B, C, H, W, dil, N, ws, st, launches);
        default: return forward_k<7>(kern, blur, sparse, conf, out, B, C, H, W, dil, N, ws, st, launches);
    }
}

int dilated2d_backward(const float* kern, const float* blur, const float* sparse, const float* conf, const float* grad_out,
                       float* grad_kern, float* grad_blur, float* grad_sparse, float* grad_conf, int B, int C, int H, int W, int K,
                       int dil, int N, void* ws, cudaStream_t st, int* launches) {
    if (N == 0) {      // d_0 = blur: the identity, and nothing reaches the weights or the samples (zero-filled by memsets)
        const size_t hw = (size_t)H * W;
        if (grad_blur) CSPN_CUDA_TRY(cudaMemcpyAsync(grad_blur, grad_out, (size_t)B * C * hw * 4, cudaMemcpyDeviceToDevice, st));
        if (grad_kern) CSPN_CUDA_TRY(cudaMemsetAsync(grad_kern, 0, (size_t)B * K * K * hw * 4, st));
        if (grad_sparse) CSPN_CUDA_TRY(cudaMemsetAsync(grad_sparse, 0, (size_t)B * hw * 4, st));
        if (grad_conf) CSPN_CUDA_TRY(cudaMemsetAsync(grad_conf, 0, (size_t)B * hw * 4, st));
        *launches = 0;
        return CSPN_OK;
    }
    switch (K) {
        case 3: return backward_k<3>(kern, blur, sparse, conf, grad_out, grad_kern, grad_blur, grad_sparse, grad_conf, B, C, H, W, dil,
                                     N, ws, st, launches);
        case 5: return backward_k<5>(kern, blur, sparse, conf, grad_out, grad_kern, grad_blur, grad_sparse, grad_conf, B, C, H, W, dil,
                                     N, ws, st, launches);
        default: return backward_k<7>(kern, blur, sparse, conf, grad_out, grad_kern, grad_blur, grad_sparse, grad_conf, B, C, H, W,
                                      dil, N, ws, st, launches);
    }
}

}  // namespace cspn
