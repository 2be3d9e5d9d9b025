// Depth metrics and the masked L1 loss ON THE DEVICE -- the consumers of the propagation's output in the reference's
// training / evaluation loops:
//   utils.evaluate_error(gt_depth, pred_depth)   /root/reference/cspn_pytorch/utils.py:19-47
//   Wighted_L1_Loss.forward(pred, label)         /root/reference/cspn_pytorch/loss.py:16-23
// The reference copies both tensors to the host after every step (train.py:204-206, eval.py:147-150) and reduces there
// with a dozen masked-select / sum calls; once the propagation itself lasts tens of microseconds that round trip is the
// step's tail (SURVEY.md 8f-4).  Here ONE pass over pred / gt produces every sum, accumulates in double, and a tiny
// finalize kernel turns them into the 12 reported numbers -- all on the caller's stream, no synchronisation.
//
// out[12] (device floats):
//   0 n_valid            4 ABS_REL            8  DELTA1.25
//   1 MSE                5 DELTA1.02          9  DELTA1.25^2
//   2 RMSE               6 DELTA1.05          10 DELTA1.25^3
//   3 MAE (== the loss)  7 DELTA1.10          11 (reserved: LG10, which the reference never fills, utils.py:23)
// Semantics follow the reference line by line: valid = gt > 0.0001 (utils.py:21, loss.py:17); diff = |gt - pred|;
// rel = diff / gt; max_ratio = max(gt / pred, pred / gt) with IEEE division (the deltas count `max_ratio < t`, so the
// quotient's rounding decides ties and must be the reference's); n_valid == 0 leaves everything 0 (utils.py:31).
// Deviations, all specified in DESIGN.md section 4.7: diff is squared and everything summed in double, and RMSE is the root
// of the double mean (the reference squares and sums in float: a diff above 1.8e19 makes its MSE and RMSE inf); out[0] is
// n_valid rounded to float, so above 2^24 the backward inverts the rounded count (at most 1 ulp in the gradient's scale);
// with n_valid == 0 the backward writes zeros, where the reference's loss is 0 / 0.
#include "common.cuh"

namespace cspn {
namespace {

constexpr int kSums = 10;   // n, sum diff^2, sum diff, sum rel, 6 delta counts

__global__ void __launch_bounds__(256)
metrics_partial_kernel(const float* __restrict__ pred, const float* __restrict__ gt, size_t n, double* __restrict__ acc) {
    double s[kSums];
#pragma unroll
    for (int i = 0; i < kSums; ++i) s[i] = 0.0;
    const float thr[6] = {1.02f, 1.05f, 1.10f, 1.25f, 1.25f * 1.25f, 1.25f * 1.25f * 1.25f};
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
        const float g = __ldg(gt + i), p = __ldg(pred + i);
        if (g > 0.0001f) {
            const float diff = fabsf(g - p);
            s[0] += 1.0;
            s[1] += (double)diff * (double)diff;
            s[2] += (double)diff;
            s[3] += (double)__fdiv_rn(diff, g);
            const float ratio = fmaxf(__fdiv_rn(g, p), __fdiv_rn(p, g));   // NaN-propagating like torch.max? see note below
#pragma unroll
            for (int t = 0; t < 6; ++t) s[4 + t] += (ratio < thr[t]) ? 1.0 : 0.0;
        }
    }
    // (torch.max propagates NaN, fmaxf drops it.  The two agree here because g / p is NaN exactly when p / g is: a NaN
    //  operand, or both infinite -- g == 0 is not valid.  Then both formulations compare NaN < t, false.  A ratio of -0 or
    //  below, from p == -0, p < 0 or p == -inf, is counted under every threshold, as the reference counts it.
    //  tests/golden/metrics/edges/ holds the reference's own results for each of these.)
#pragma unroll
    for (int i = 0; i < kSums; ++i) {
        double v = s[i];
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
        s[i] = v;
    }
    __shared__ double sh[8][kSums];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    if (lane == 0)
#pragma unroll
        for (int i = 0; i < kSums; ++i) sh[warp][i] = s[i];
    __syncthreads();
    if (threadIdx.x < kSums) {
        double v = 0.0;
        for (int w = 0; w < 8; ++w) v += sh[w][threadIdx.x];
        atomicAdd(acc + threadIdx.x, v);
    }
}

__global__ void metrics_finalize_kernel(const double* __restrict__ acc, float* __restrict__ out) {
    if (threadIdx.x != 0) return;
    const double n = acc[0];
    for (int i = 0; i < 12; ++i) out[i] = 0.f;
    out[0] = (float)n;
    if (n > 0.0) {
        const double mse = acc[1] / n;
        out[1] = (float)mse;
        out[2] = (float)sqrt(mse);
        out[3] = (float)(acc[2] / n);
        out[4] = (float)(acc[3] / n);
        for (int t = 0; t < 6; ++t) out[5 + t] = (float)(acc[4 + t] / n);
    }
}

__global__ void __launch_bounds__(256)
masked_l1_bwd_kernel(const float* __restrict__ pred, const float* __restrict__ gt, const float* __restrict__ stats,
                     const float* __restrict__ grad_loss, float* __restrict__ grad_pred, size_t n) {
    const float nv = __ldg(stats);                              // n_valid
    const float scale = (nv > 0.f ? 1.f / nv : 0.f) * (grad_loss ? __ldg(grad_loss) : 1.f);
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
        const float g = __ldg(gt + i), d = __ldg(pred + i) - g;
        // d/dpred |pred - label| = sign(pred - label) (0 at the kink, as torch.abs' backward), only where label is valid
        grad_pred[i] = (g > 0.0001f) ? scale * ((d > 0.f ? 1.f : 0.f) - (d < 0.f ? 1.f : 0.f)) : 0.f;
    }
}

int grid_for(size_t n) {
    size_t b = (n + 255) / 256;
    const size_t cap = 132 * 8;   // 8 blocks per SM of an H100 SXM
    return (int)(b < 1 ? 1 : (b > cap ? cap : b));
}

}  // namespace
}  // namespace cspn

using namespace cspn;

extern "C" {

CSPN_API size_t cspn_depth_metrics_workspace_bytes(void) { return kSums * sizeof(double); }

CSPN_API int cspn_depth_metrics_f32(const float* pred, const float* gt, size_t n, float* out12, void* workspace, size_t workspace_bytes,
                           cspn_stream_t stream) {
    clear_error();
    if (!pred || !gt || !out12) { set_error("null tensor pointer"); return CSPN_ERR_INVALID_ARGUMENT; }
    if (!workspace || workspace_bytes < kSums * sizeof(double) || (reinterpret_cast<uintptr_t>(workspace) & 7)) {
        set_error("depth metrics need %zu bytes of 8-byte aligned workspace", kSums * sizeof(double));
        return CSPN_ERR_WORKSPACE;
    }
    cudaStream_t st = (cudaStream_t)stream;
    double* acc = static_cast<double*>(workspace);
    CSPN_CUDA_TRY(cudaMemsetAsync(acc, 0, kSums * sizeof(double), st));
    if (n > 0) metrics_partial_kernel<<<grid_for(n), 256, 0, st>>>(pred, gt, n, acc);
    metrics_finalize_kernel<<<1, 32, 0, st>>>(acc, out12);
    CSPN_CUDA_TRY(cudaGetLastError());
    return CSPN_OK;
}

CSPN_API int cspn_masked_l1_bwd_f32(const float* pred, const float* gt, const float* stats12, const float* grad_loss, float* grad_pred,
                           size_t n, cspn_stream_t stream) {
    clear_error();
    if (!pred || !gt || !stats12 || !grad_pred) { set_error("null tensor pointer"); return CSPN_ERR_INVALID_ARGUMENT; }
    if (n > 0) masked_l1_bwd_kernel<<<grid_for(n), 256, 0, (cudaStream_t)stream>>>(pred, gt, stats12, grad_loss, grad_pred, n);
    CSPN_CUDA_TRY(cudaGetLastError());
    return CSPN_OK;
}

}  // extern "C"
