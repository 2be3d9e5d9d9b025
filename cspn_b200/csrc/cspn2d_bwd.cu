// 2D CSPN backward: the adjoint of cspn2d forward, for training through the operator
// (reference: autograd through /root/reference/cspn_pytorch/models/cspn.py:42-144 as used by train.py:196-199).
//
// Forward (folded form, see cspn2d_generic.cu):  w'_k = (1-m) a_k / S,  kappa = (1-m)(1 - A/S) + m,  c' = kappa d0,
//     d_{t+1} = c' + sum_k w'_k shift_k(d_t),   a_k(p) = ghat_k(p + off_k),  S = sum|a_k|,  A = sum a_k,  m = sign(sparse).
// Backward, with lambda_N = grad_out:
//     lambda_t(q)   = sum_k w'_k(q - off_k) lambda_{t+1}(q - off_k)                (adjoint stencil, gather form)
//     Gw_k(p)      += sum_c lambda_{t+1,c}(p) d_{t,c}(p + off_k)                   (dL/dw'_k, summed over steps/channels)
//     Gc_c(p)      += lambda_{t+1,c}(p)                                            (dL/dc')
// then through the folding and the normalisation (om = 1 - m, w_k = a_k / S):
//     Gkappa = sum_c Gc_c d0_c,   H_k = om (Gw_k - Gkappa) = dL/dw_k,   T = sum_k H_k w_k,
//     dL/da_j = (H_j - sign(a_j) T) / S,   grad_g_j(p + off_j) = dL/da_j(p) [* sign(g_j) in '8sum_abs'],
//     grad_blur_c = kappa Gc_c + lambda_{0,c}.
// Every g_j(q) feeds exactly one pixel (p = q - off_j), so the scatter into grad_guidance needs no atomics.
// The forward iterates d_1..d_{N-1} are recomputed and kept in the workspace ((N-1) B C H W floats).
//
// Two formulations:
//  * cluster (default; checked against fp64 autograd through the reference's op sequence and the gradient goldens): the forward cluster kernel in kStoreSteps mode writes every iterate, the same kernel in kAdjoint
//    mode runs the transposed stencil register-resident and writes every lambda_t, and one gather kernel forms
//    Gw_k(p) = sum_t lambda_{t+1}(p) d_t(p + off_k), Gc = sum_t lambda_{t+1} straight into the finalize arithmetic:
//    no Gw planes in memory, 2 N planes of workspace.
//  * launch-per-step (W % 4 != 0, misaligned tensors, or CSPN_B200_BWD=steps): generic prep + N-1 forward steps, N adjoint
//    steps that also read-modify-write the 8 planes of Gw, finalize.
#include <cstdlib>
#include <cstring>

#include "common.cuh"

namespace cspn {

namespace {

// one backward step: reads lambda_{t+1} (lam_in), d_t; writes lambda_t (lam_out); accumulates Gw, Gc
__global__ void __launch_bounds__(256)
bwd_step_kernel(const float* __restrict__ wk, const float* __restrict__ d_t, const float* __restrict__ lam_in,
                float* __restrict__ lam_out, float* __restrict__ Gw, float* __restrict__ Gc, int C, int H, int W,
                int first) {
    const int x = blockIdx.x * blockDim.x + threadIdx.x;
    const int y = blockIdx.y * blockDim.y + threadIdx.y;
    const int b = blockIdx.z;
    if (x >= W || y >= H) return;
    const size_t HW = (size_t)H * W, p = (size_t)y * W + x;
    const float* w = wk + (size_t)b * 9 * HW;
    float gw[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) gw[k] = first ? 0.f : Gw[((size_t)b * 8 + k) * HW + p];
    for (int c = 0; c < C; ++c) {
        const size_t plane = ((size_t)b * C + c) * HW;
        const float* li = lam_in + plane;
        const float* dt = d_t + plane;
        const float lp = __ldg(li + p);
        float acc = 0.f;
#pragma unroll
        for (int k = 0; k < 8; ++k) {
            // destination pixel (y - dy, x - dx) reads this pixel with tap k
            const int ys = y - off2_dy(k), xs = x - off2_dx(k);
            if (ys >= 0 && ys < H && xs >= 0 && xs < W) {
                const size_t ps = (size_t)ys * W + xs;
                acc = fmaf(__ldg(w + k * HW + ps), __ldg(li + ps), acc);
            }
            const int yn = y + off2_dy(k), xn = x + off2_dx(k);
            if (yn >= 0 && yn < H && xn >= 0 && xn < W) gw[k] = fmaf(lp, __ldg(dt + (size_t)yn * W + xn), gw[k]);
        }
        lam_out[plane + p] = acc;
        Gc[plane + p] = (first ? 0.f : Gc[plane + p]) + lp;
    }
#pragma unroll
    for (int k = 0; k < 8; ++k) Gw[((size_t)b * 8 + k) * HW + p] = gw[k];
}

__global__ void __launch_bounds__(256)
bwd_finalize_kernel(const float* __restrict__ guidance, const float* __restrict__ blur, const float* __restrict__ sparse,
                    const float* __restrict__ wk, const float* __restrict__ Gw, const float* __restrict__ Gc,
                    const float* __restrict__ lam0, float* __restrict__ grad_guidance, float* __restrict__ grad_blur, int C,
                    int H, int W, int gch, int norm_abs) {
    const int x = blockIdx.x * blockDim.x + threadIdx.x;
    const int y = blockIdx.y * blockDim.y + threadIdx.y;
    const int b = blockIdx.z;
    if (x >= W || y >= H) return;
    const size_t HW = (size_t)H * W, p = (size_t)y * W + x;
    const float kappa = __ldg(wk + ((size_t)b * 9 + 8) * HW + p);
    float gkappa = 0.f;
    for (int c = 0; c < C; ++c) {
        const size_t plane = ((size_t)b * C + c) * HW;
        const float gc = __ldg(Gc + plane + p);
        gkappa = fmaf(gc, __ldg(blur + plane + p), gkappa);
        if (grad_blur) grad_blur[plane + p] = fmaf(kappa, gc, __ldg(lam0 + plane + p));
    }
    if (!grad_guidance) return;
    const float* g = guidance + (size_t)b * gch * HW;
    float a[8], sg[8], S = 0.f;
#pragma unroll
    for (int k = 0; k < 8; ++k) {
        const int yy = y + off2_dy(k), xx = x + off2_dx(k);
        float v = 0.f;
        sg[k] = 1.f;
        if (yy >= 0 && yy < H && xx >= 0 && xx < W) {
            v = __ldg(g + k * HW + (size_t)yy * W + xx);
            if (norm_abs) { sg[k] = signf(v); v = fabsf(v); }   // d|g|/dg = sign(g) (0 at 0, like torch.abs)
        }
        a[k] = v;
        S += fabsf(v);
    }
    const float m = sparse ? signf(__ldg(sparse + (size_t)b * HW + p)) : 0.f;
    const float om = 1.f - m;
    float Hk[8], T = 0.f;
#pragma unroll
    for (int k = 0; k < 8; ++k) {
        Hk[k] = om * (__ldg(Gw + ((size_t)b * 8 + k) * HW + p) - gkappa);
        T = fmaf(Hk[k], __fdiv_rn(a[k], S), T);
    }
#pragma unroll
    for (int k = 0; k < 8; ++k) {
        const int yy = y + off2_dy(k), xx = x + off2_dx(k);
        if (yy >= 0 && yy < H && xx >= 0 && xx < W) {
            const float ga = __fdiv_rn(Hk[k] - signf(a[k]) * T, S);
            grad_guidance[((size_t)b * gch + k) * HW + (size_t)yy * W + xx] = ga * sg[k];
        }
    }
}

// Staged cluster formulation, last stage: Gw / Gc gathered over all steps in registers, then the finalize arithmetic
// of bwd_finalize_kernel.  steps[t] = d_{t+1}, lam[t] = lambda_t (planes of n = B*C*H*W floats), lambda_N = grad_out.
__global__ void __launch_bounds__(256)
bwd_gather_finalize_kernel(const float* __restrict__ guidance, const float* __restrict__ blur, const float* __restrict__ sparse,
                           const float* __restrict__ steps, const float* __restrict__ lam, const float* __restrict__ grad_out,
                           float* __restrict__ grad_guidance, float* __restrict__ grad_blur, long long n, int N, int C, int H,
                           int W, int gch, int norm_abs) {
    const int x = blockIdx.x * blockDim.x + threadIdx.x;
    const int y = blockIdx.y * blockDim.y + threadIdx.y;
    const int b = blockIdx.z;
    if (x >= W || y >= H) return;
    const size_t HW = (size_t)H * W, p = (size_t)y * W + x;
    const float* g = guidance + (size_t)b * gch * HW;
    float a[8], sg[8], S = 0.f;
    bool nb_in[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) {
        const int yy = y + off2_dy(k), xx = x + off2_dx(k);
        nb_in[k] = yy >= 0 && yy < H && xx >= 0 && xx < W;
        float v = 0.f;
        sg[k] = 1.f;
        if (nb_in[k]) {
            v = __ldg(g + k * HW + (size_t)yy * W + xx);
            if (norm_abs) { sg[k] = signf(v); v = fabsf(v); }
        }
        a[k] = v;
        S += fabsf(v);
    }
    const float m = sparse ? signf(__ldg(sparse + (size_t)b * HW + p)) : 0.f;
    const float om = 1.f - m;
    float wsum = 0.f;
#pragma unroll
    for (int k = 0; k < 8; ++k) wsum += __fdiv_rn(a[k], S);
    const float kappa = om * (1.f - wsum) + m;

    float gw[8], gkappa = 0.f;
#pragma unroll
    for (int k = 0; k < 8; ++k) gw[k] = 0.f;
    for (int c = 0; c < C; ++c) {
        const size_t plane = ((size_t)b * C + c) * HW;
        float gc = 0.f;
        for (int t = 0; t < N; ++t) {
            const float lp = __ldg((t == N - 1 ? grad_out : lam + (size_t)(t + 1) * n) + plane + p);
            const float* dt = (t == 0 ? blur : steps + (size_t)(t - 1) * n) + plane;
            gc += lp;
#pragma unroll
            for (int k = 0; k < 8; ++k)
                if (nb_in[k]) gw[k] = fmaf(lp, __ldg(dt + (size_t)(y + off2_dy(k)) * W + (x + off2_dx(k))), gw[k]);
        }
        gkappa = fmaf(gc, __ldg(blur + plane + p), gkappa);
        if (grad_blur) grad_blur[plane + p] = fmaf(kappa, gc, __ldg(lam + plane + p));   // lam[0] = lambda_0
    }
    if (!grad_guidance) return;
    float Hk[8], T = 0.f;
#pragma unroll
    for (int k = 0; k < 8; ++k) {
        Hk[k] = om * (gw[k] - gkappa);
        T = fmaf(Hk[k], __fdiv_rn(a[k], S), T);
    }
#pragma unroll
    for (int k = 0; k < 8; ++k)
        if (nb_in[k]) {
            const float ga = __fdiv_rn(Hk[k] - signf(a[k]) * T, S);
            grad_guidance[((size_t)b * gch + k) * HW + (size_t)(y + off2_dy(k)) * W + (x + off2_dx(k))] = ga * sg[k];
        }
}

// The register-resident formulation is the default; CSPN_B200_BWD=steps forces the launch-per-step one (cross-check in
// tests/test_cluster_backward_gpu.py, and the path shapes outside the cluster kernel's take anyway).
bool cluster_backward_enabled() {
    const char* e = getenv("CSPN_B200_BWD");
    return !(e && strcmp(e, "steps") == 0);
}

}  // namespace

size_t bwd2d_workspace_bytes(int B, int C, int H, int W, int iters) {
    if (iters <= 0) return 0;
    const size_t HW = (size_t)H * W, n = (size_t)B * C * HW;
    // wk (9 planes/image) + d_1..d_{N-1} + lambda ping-pong + Gw + Gc
    const size_t per_step = sizeof(float) * ((size_t)B * 9 * HW + (size_t)(iters - 1) * n + 2 * n + (size_t)B * 8 * HW + n);
    const size_t cluster = cluster_backward_enabled() ? sizeof(float) * 2 * (size_t)iters * n : 0;   // d_1..d_N, lambda_0..lambda_{N-1}
    return per_step > cluster ? per_step : cluster;
}

// Cluster formulation (see the file header).  Returns CSPN_ERR_UNSUPPORTED when the shape / alignment is not
// the cluster kernel's; the caller then falls back to the launch-per-step path.
static int bwd2d_cluster(const Problem2D& p, const float* grad_out, float* grad_guidance, float* grad_blur, void* ws,
                         cudaStream_t stream, int* launches) {
    char why[200] = "";
    if ((reinterpret_cast<uintptr_t>(grad_out) | reinterpret_cast<uintptr_t>(ws)) & 15) return CSPN_ERR_UNSUPPORTED;
    if (!cluster2d_supported(p, why, sizeof(why))) return CSPN_ERR_UNSUPPORTED;
    const long long n = (long long)p.B * p.C * p.H * p.W;
    float* steps = static_cast<float*>(ws);            // steps[t] = d_{t+1}
    float* lam = steps + (size_t)p.iters * n;          // lam[t]   = lambda_t
    int rc = cluster2d_forward_steps(p, steps, stream, launches);
    if (rc != CSPN_OK) return rc;
    rc = cluster2d_adjoint_steps(p, grad_out, lam, stream, launches);
    if (rc != CSPN_OK) return rc;
    const dim3 block(32, 8);
    const dim3 grid((p.W + 31) / 32, (p.H + 7) / 8, p.B);
    bwd_gather_finalize_kernel<<<grid, block, 0, stream>>>(p.guidance, p.blur, p.sparse, steps, lam, grad_out, grad_guidance,
                                                            grad_blur, n, p.iters, p.C, p.H, p.W, p.gch, p.norm_abs);
    ++*launches;
    CSPN_CUDA_TRY(cudaGetLastError());
    return CSPN_OK;
}

int bwd2d(const Problem2D& p, const float* grad_out, float* grad_guidance, float* grad_blur, void* ws, size_t ws_bytes,
          cudaStream_t stream, int* launches) {
    const size_t HW = (size_t)p.H * p.W, n = (size_t)p.B * p.C * HW;
    if (grad_guidance)
        CSPN_CUDA_TRY(cudaMemsetAsync(grad_guidance, 0, (size_t)p.B * p.gch * HW * sizeof(float), stream));
    if (p.iters == 0) {
        if (grad_blur) CSPN_CUDA_TRY(cudaMemcpyAsync(grad_blur, grad_out, n * sizeof(float), cudaMemcpyDeviceToDevice, stream));
        return CSPN_OK;
    }
    const size_t need = bwd2d_workspace_bytes(p.B, p.C, p.H, p.W, p.iters);
    if (!ws || ws_bytes < need) {
        set_error("2D backward needs %zu workspace bytes, got %zu", need, ws ? ws_bytes : (size_t)0);
        return CSPN_ERR_WORKSPACE;
    }
    if (p.B > 65535 || (long)p.B * p.C > 65535) { set_error("backward: B*C exceeds gridDim.z"); return CSPN_ERR_UNSUPPORTED; }
    if (cluster_backward_enabled()) {
        const int rc = bwd2d_cluster(p, grad_out, grad_guidance, grad_blur, ws, stream, launches);
        if (rc != CSPN_ERR_UNSUPPORTED) return rc;
        clear_error();   // shape / alignment outside the cluster kernel's: the launch-per-step path below handles it
    }
    float* wk = static_cast<float*>(ws);
    float* D = wk + (size_t)p.B * 9 * HW;             // d_1 .. d_{N-1}
    float* lam[2] = {D + (size_t)(p.iters - 1) * n, D + (size_t)(p.iters - 1) * n + n};
    float* Gw = lam[1] + n;
    float* Gc = Gw + (size_t)p.B * 8 * HW;

    launch_prep2d(p.guidance, p.sparse, wk, p.B, p.H, p.W, p.gch, p.norm_abs, stream);
    ++*launches;
    for (int t = 0; t + 1 < p.iters; ++t) {           // d_{t+1} = step(d_t)
        launch_step2d(wk, p.blur, t == 0 ? p.blur : D + (size_t)(t - 1) * n, D + (size_t)t * n, p.B, p.C, p.H, p.W, stream);
        ++*launches;
    }
    const dim3 block(32, 8);
    const dim3 grid((p.W + 31) / 32, (p.H + 7) / 8, p.B);
    const float* lam_in = grad_out;
    for (int t = p.iters - 1; t >= 0; --t) {
        float* lam_out = lam[t & 1];
        const float* d_t = (t == 0) ? p.blur : D + (size_t)(t - 1) * n;
        bwd_step_kernel<<<grid, block, 0, stream>>>(wk, d_t, lam_in, lam_out, Gw, Gc, p.C, p.H, p.W, t == p.iters - 1);
        ++*launches;
        lam_in = lam_out;
    }
    bwd_finalize_kernel<<<grid, block, 0, stream>>>(p.guidance, p.blur, p.sparse, wk, Gw, Gc, lam_in, grad_guidance, grad_blur,
                                                    p.C, p.H, p.W, p.gch, p.norm_abs);
    ++*launches;
    CSPN_CUDA_TRY(cudaGetLastError());
    return CSPN_OK;
}

}  // namespace cspn
