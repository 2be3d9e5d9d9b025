// Generic 2D CSPN forward: one "prep" launch (affinity normalisation + mask folding) and one
// 9-point stencil launch per iteration.  Handles every shape (odd W, huge H, prop_time of any
// size); it is the forward fallback of the cluster kernel (cspn2d_cluster.cu) and the simplest
// statement of the arithmetic on the GPU.  The fallback backward is the K x K one of cspn2d_wide.cu
// at K = 3 (cspn2d_bwd.cu): the 3x3 step there measured slower on odd widths (DESIGN.md section 4.8).
//
// Arithmetic (SURVEY.md Appendix A; reference /root/reference/cspn_pytorch/models/cspn.py):
//   a_k(p) = g_k(p + off_k) (0 outside the image)             cspn.py:105-132
//   w_k    = a_k / sum_j |a_j|,   s = sum_k w_k               cspn.py:135-142
//   m      = sign(sparse)                                     cspn.py:63-64
//   folded: w'_k = (1-m) w_k,  kappa = (1-m)(1-s) + m   so that one iteration
//   d <- (1-m)[(1-s) d0 + sum_k w_k shift_k(d)] + m d0        cspn.py:70-81
//   becomes d <- kappa*d0 + sum_k w'_k shift_k(d).
// Workspace: B*9*H*W floats (w'_0..7, kappa; shared by the C channels) + B*C*H*W (ping-pong).
#include "common.cuh"

namespace cspn {

namespace {

__global__ void __launch_bounds__(256)
prep2d_kernel(const float* __restrict__ guidance, const float* __restrict__ sparse, float* __restrict__ wk,
              int H, int W, int gch, int norm_abs) {
    const int x = blockIdx.x * blockDim.x + threadIdx.x;
    const int y = blockIdx.y * blockDim.y + threadIdx.y;
    const int b = blockIdx.z;
    if (x >= W || y >= H) return;
    const size_t HW = (size_t)H * W;
    const float* g = guidance + (size_t)b * gch * HW;
    float a[8], S = 0.f;
#pragma unroll
    for (int k = 0; k < 8; ++k) {
        const int yy = y + off2_dy(k), xx = x + off2_dx(k);
        float v = 0.f;
        if (yy >= 0 && yy < H && xx >= 0 && xx < W) {
            v = __ldg(g + k * HW + (size_t)yy * W + xx);
            if (norm_abs) v = fabsf(v);
        }
        a[k] = v;
        S += fabsf(v);
    }
    const size_t p = (size_t)y * W + x;
    const float m = sparse ? signf(__ldg(sparse + (size_t)b * HW + p)) : 0.f;
    const float om = 1.f - m;
    float s = 0.f;
    float* o = wk + (size_t)b * 9 * HW + p;
#pragma unroll
    for (int k = 0; k < 8; ++k) {
        const float w = __fdiv_rn(a[k], S);  // IEEE: 0/0 -> NaN like torch.div (cspn.py:138)
        s += w;
        o[k * HW] = om * w;
    }
    o[8 * HW] = om * (1.f - s) + m;
}

__global__ void __launch_bounds__(256)
step2d_kernel(const float* __restrict__ wk, const float* __restrict__ d0, const float* __restrict__ cur,
              float* __restrict__ dst, int C, int H, int W) {
    const int x = blockIdx.x * blockDim.x + threadIdx.x;
    const int y = blockIdx.y * blockDim.y + threadIdx.y;
    const int bc = blockIdx.z;
    if (x >= W || y >= H) return;
    const size_t HW = (size_t)H * W;
    const size_t p = (size_t)y * W + x;
    const float* w = wk + (size_t)(bc / C) * 9 * HW + p;
    const float* c = cur + (size_t)bc * HW;
    float acc = __ldg(w + 8 * HW) * __ldg(d0 + (size_t)bc * HW + p);
#pragma unroll
    for (int k = 0; k < 8; ++k) {
        const int yy = y + off2_dy(k), xx = x + off2_dx(k);
        const float dv = (yy >= 0 && yy < H && xx >= 0 && xx < W) ? __ldg(c + (size_t)yy * W + xx) : 0.f;
        acc = fmaf(__ldg(w + k * HW), dv, acc);
    }
    dst[(size_t)bc * HW + p] = acc;
}

}  // namespace

// keep: the d0' planes of the keep-sparse mode follow the ping-pong buffer
size_t generic2d_workspace_bytes(int B, int C, int H, int W, int iters, bool keep) {
    if (iters <= 0) return 0;
    const size_t HW = (size_t)H * W;
    return sizeof(float) * ((size_t)B * 9 * HW + (iters > 1 ? (size_t)B * C * HW : 0) + (keep ? (size_t)B * C * HW : 0));
}

int generic2d_forward(const Problem2D& p, void* ws, size_t ws_bytes, cudaStream_t stream, int* launches) {
    const size_t HW = (size_t)p.H * p.W;
    const size_t n = (size_t)p.B * p.C * HW;
    if (p.iters == 0) {
        CSPN_CUDA_TRY(cudaMemcpyAsync(p.out, p.blur, n * sizeof(float), cudaMemcpyDeviceToDevice, stream));
        return CSPN_OK;
    }
    const size_t need = generic2d_workspace_bytes(p.B, p.C, p.H, p.W, p.iters, p.keep);
    if (!ws || ws_bytes < need) {
        set_error("generic 2D path needs %zu workspace bytes, got %zu", need, ws ? ws_bytes : (size_t)0);
        return CSPN_ERR_WORKSPACE;
    }
    float* wk = static_cast<float*>(ws);
    float* tmp = wk + (size_t)p.B * 9 * HW;
    const dim3 block(32, 8);
    const dim3 gx((p.W + 31) / 32, (p.H + 7) / 8);
    if (p.B > 65535 || p.B * p.C > 65535) {
        set_error("generic 2D path: B*C=%d exceeds gridDim.z", p.B * p.C);
        return CSPN_ERR_UNSUPPORTED;
    }
    // keep-sparse mode: the same step kernel, its constant term kappa * d0 reading d0' = (1-m) blur + m sparse
    const float* d0 = p.blur;
    if (p.keep) {
        float* d0k = tmp + (p.iters > 1 ? n : 0);
        launch_prep_keep(3, p.guidance, p.sparse, p.blur, wk, d0k, p.B, p.C, p.H, p.W, p.gch, p.norm_abs, stream);
        d0 = d0k;
    } else {
        prep2d_kernel<<<dim3(gx.x, gx.y, p.B), block, 0, stream>>>(p.guidance, p.sparse, wk, p.H, p.W, p.gch,
                                                                    p.norm_abs);
    }
    ++*launches;
    // ping-pong so that the last iteration writes p.out
    const float* cur = p.blur;
    float* dst = (p.iters & 1) ? p.out : tmp;
    for (int it = 0; it < p.iters; ++it) {
        step2d_kernel<<<dim3(gx.x, gx.y, p.B * p.C), block, 0, stream>>>(wk, d0, cur, dst, p.C, p.H, p.W);
        ++*launches;
        cur = dst;
        dst = (dst == p.out) ? tmp : p.out;
    }
    CSPN_CUDA_TRY(cudaGetLastError());
    return CSPN_OK;
}

}  // namespace cspn
