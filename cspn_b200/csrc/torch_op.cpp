// torch.ops.cspn_b200.* -- the PyTorch operator registration of the CSPN propagation path.
//
// A thin C++ shim over the C ABI of include/cspn_b200.h (libcspn_b200.so): PyTorch supplies device memory, the current
// stream and the dispatcher entry; every byte of arithmetic stays in the hand-written sm_90a kernels.  Registered as
// dispatcher ops (TORCH_LIBRARY) so that torch.compile / torch.export trace the call the reference model makes at
// /root/reference/cspn_pytorch/models/torch_resnet_cspn_nyu.py:375 as ONE opaque node; the fake (meta) kernels and the
// autograd formulas are registered from Python (cspn_b200/torch_op.py) with torch.library.
//
// Schema (norm_type / algo are the enums of include/cspn_b200.h):
//   propagate2d(Tensor guidance, Tensor blur_depth, Tensor? sparse_depth, int prop_time, int norm_type, int algo) -> Tensor
//   propagate2d_backward(Tensor guidance, Tensor blur_depth, Tensor? sparse_depth, Tensor grad_out, int prop_time,
//                        int norm_type, bool need_guidance, bool need_blur) -> (Tensor, Tensor)
//   propagate2d_k(Tensor guidance, Tensor blur_depth, Tensor? sparse_depth, int kernel_size, int prop_time, int norm_type)
//       -> Tensor                                                    (K x K kernel, K in {3, 5, 7}; K = 3 is propagate2d)
//   propagate2d_k_backward(Tensor guidance, Tensor blur_depth, Tensor? sparse_depth, Tensor grad_out, int kernel_size,
//                          int prop_time, int norm_type, bool need_guidance, bool need_blur) -> (Tensor, Tensor)
//   propagate2d_keep(Tensor guidance, Tensor blur_depth, Tensor? sparse_depth, int kernel_size, int prop_time, int norm_type,
//                    int algo) -> Tensor           (keep-sparse mode: the samples stay in the output, K in {3, 5, 7})
//   propagate2d_keep_backward(Tensor guidance, Tensor blur_depth, Tensor? sparse_depth, Tensor grad_out, int kernel_size,
//                             int prop_time, int norm_type, bool need_guidance, bool need_blur, bool need_sparse)
//       -> (Tensor, Tensor, Tensor)
//   propagate2d_aggregate(Tensor guidance, Tensor blur_depth, Tensor? sparse_depth, Tensor step_weight, int[] steps,
//                         int kernel_size, int norm_type, bool keep) -> Tensor
//       (CSPN++'s context-aware CSPN: sum_j step_weight[:, j] * d_{steps[j]}, K in {3, 5, 7}, keep the keep-sparse mode)
//   propagate2d_aggregate_backward(Tensor guidance, Tensor blur_depth, Tensor? sparse_depth, Tensor step_weight,
//                                  Tensor grad_out, int[] steps, int kernel_size, int norm_type, bool keep,
//                                  bool need_guidance, bool need_blur, bool need_sparse, bool need_step_weight)
//       -> (Tensor, Tensor, Tensor, Tensor)
//   propagate2d_nonlocal(Tensor feat, Tensor offset, Tensor affinity, Tensor? sparse_depth, int kernel_size, int prop_time)
//       -> Tensor   (NLSPN's non-local propagation: offset (B, 2T, H, W), affinity (B, T, H, W), T = K*K-1, K in {3, 5, 7})
//   propagate2d_nonlocal_backward(Tensor feat, Tensor offset, Tensor affinity, Tensor? sparse_depth, Tensor grad_out,
//                                 int kernel_size, int prop_time, bool need_feat, bool need_offset, bool need_affinity,
//                                 bool need_sparse) -> (Tensor, Tensor, Tensor, Tensor)
//   propagate2d_dilated(Tensor kernel, Tensor blur_depth, Tensor? sparse_depth, Tensor? confidence, int kernel_size,
//                       int dilation, int prop_time) -> Tensor   (PENet's DA-CSPN++ step: kernel (B, K*K, H, W), sparse_depth
//                       and confidence (B, 1, H, W), both or neither, K in {3, 5, 7}, dilation in [1, 4])
//   propagate2d_dilated_backward(Tensor kernel, Tensor blur_depth, Tensor? sparse_depth, Tensor? confidence, Tensor grad_out,
//                                int kernel_size, int dilation, int prop_time, bool need_kernel, bool need_blur,
//                                bool need_sparse, bool need_confidence) -> (Tensor, Tensor, Tensor, Tensor)
//   propagate2d_dynamic(Tensor affinity, Tensor attention, Tensor blur_depth, Tensor? sparse_depth, Tensor? confidence,
//                       int kernel_size) -> Tensor   (DySPN's step: affinity (B, K*K, H, W), attention (B, N*(K+1)/2, H, W),
//                       sparse_depth and confidence (B, 1, H, W), both or neither, K in {3, 5, 7})
//   propagate2d_dynamic_backward(Tensor affinity, Tensor attention, Tensor blur_depth, Tensor? sparse_depth, Tensor? confidence,
//                                Tensor grad_out, int kernel_size, bool need_affinity, bool need_attention, bool need_blur,
//                                bool need_sparse, bool need_confidence) -> (Tensor, Tensor, Tensor, Tensor, Tensor)
//   propagate2d_linear(Tensor feat, Tensor gate, int dir_mask) -> (Tensor, Tensor)
//       (SPN's three-way scans: feat (B, C, H, W), gate (B, 3*nd, H, W) shared or (B, 3*nd*C, H, W) per channel with C > 1,
//       dir_mask bits l2r, r2l, t2b, b2t; returns the merged output and the per-direction planes (nd, B, C, H, W), empty
//       for nd = 1)
//   propagate2d_linear_backward(Tensor feat, Tensor gate, Tensor planes, Tensor grad_out, int dir_mask, bool need_feat,
//                               bool need_gate) -> (Tensor, Tensor)   (planes: the forward's planes, its output for nd = 1)
//   propagate2d_paddle(Tensor guidance, Tensor feat, int kernel_size, int prop_time) -> Tensor
//       (own-location gates, K in {3, 5, 7}; guidance (B, K*K-1, H, W) shared, or (B, (K*K-1)*C, H, W) per channel)
//   propagate2d_paddle_backward(Tensor guidance, Tensor feat, Tensor grad_out, int kernel_size, int prop_time,
//                               bool need_guidance, bool need_feat) -> (Tensor, Tensor)
//   propagate3d(Tensor guidance, Tensor feat, int prop_time, int norm_type) -> Tensor
//   propagate3d_backward(Tensor guidance, Tensor feat, Tensor grad_out, int prop_time, int norm_type,
//                        bool need_guidance, bool need_feat) -> (Tensor, Tensor)
//   propagate3d_k(Tensor guidance, Tensor feat, int kernel_size, int prop_time, int norm_type) -> Tensor
//       (K x K x K kernel, K in {3, 5}; K = 3 is propagate3d)
//   propagate3d_k_backward(Tensor guidance, Tensor feat, Tensor grad_out, int kernel_size, int prop_time, int norm_type,
//                          bool need_guidance, bool need_feat) -> (Tensor, Tensor)
//   affinity_propagate2d(Tensor input, Tensor gate_weight, int kernel_size, int prop_step) -> Tensor
//       (fluid.layers.affinity_propagate with the caller's gates, K in {3, 5, 7}; gate_weight (B, K*K-1, H, W) shared, or
//       (B, (K*K-1)*C, H, W) per channel)
//   affinity_propagate2d_backward(Tensor input, Tensor gate_weight, Tensor grad_out, int kernel_size, int prop_step,
//                                 bool need_input, bool need_gate) -> (Tensor, Tensor)
//   affinity_propagate3d / affinity_propagate3d_backward: the same for (B, C, D, H, W), K in {3, 5}
//   unpool_conv3x3(Tensor x, Tensor weight, int H, int W) -> Tensor
//       (the guidance / depth head: Unpool, crop to H x W, 3x3 convolution; x (B, Cin, h, w), weight (Cout, Cin, 3, 3))
//   unpool_conv3x3_backward(Tensor x, Tensor weight, Tensor grad_out, int H, int W, bool need_x, bool need_weight)
//       -> (Tensor, Tensor)
//   resize_trilinear(Tensor input, int D, int H, int W, bool align_corners, int align_mode) -> Tensor
//       (fluid.layers.resize_trilinear: input (B, C, d, h, w) resampled to (B, C, D, H, W))
//   resize_trilinear_backward(Tensor grad_out, int in_D, int in_H, int in_W, bool align_corners, int align_mode) -> Tensor
//       (grad_input (B, C, in_D, in_H, in_W) from grad_out alone: the backward needs the input's size only)
//   disparity_regression(Tensor cost, int D, int H, int W, bool align_corners, int align_mode) -> Tensor
//       (cost (B, C, d, h, w) resized to (D, H, W), softmax over D, expectation of the index: (B, C, H, W))
//   disparity_regression_backward(Tensor cost, Tensor grad_out, int D, int H, int W, bool align_corners, int align_mode)
//       -> Tensor   (grad_cost (B, C, d, h, w); the softmax is recomputed from cost)
//   concat_volume(Tensor left, Tensor right, int max_disp) -> Tensor
//       (PSMNet's concatenation volume: left, right (B, F, H, W) -> (B, 2F, max_disp, H, W))
//   concat_volume_backward(Tensor grad_out) -> (Tensor, Tensor)      (grad_left, grad_right from grad_out alone)
//   gwc_volume(Tensor left, Tensor right, int max_disp, int num_groups) -> Tensor
//       (GwcNet's group-wise correlation volume: (B, F, H, W) -> (B, num_groups, max_disp, H, W))
//   gwc_volume_backward(Tensor left, Tensor right, Tensor grad_out) -> (Tensor, Tensor)
//   affinity_pool2d(Tensor feat, Tensor gate, int[] kernel_sizes) -> Tensor
//       (CSPN's spatial pyramid pooling: feat (B, C, H, W) and gate (B, L, H, W) -> the L levels (B, C, H/p, W/p) packed
//       level-major in one flat tensor)
//   affinity_pool2d_backward(Tensor feat, Tensor gate, Tensor out, Tensor grad_out, int[] kernel_sizes) -> (Tensor, Tensor)
//       (grad_feat, grad_gate; out and grad_out packed as the forward's result)
//   affinity_fuse2d(Tensor[] levels, Tensor gate, bool align_corners, int align_mode) -> Tensor
//       (CSPN's spatial pyramid fusion: L levels (B, C, h_l, w_l) upsampled to gate (B, L, H, W)'s size and combined with
//       its normalised affinities -> (B, C, H, W))
//   affinity_fuse2d_backward(Tensor[] levels, Tensor gate, Tensor out, Tensor grad_out, bool align_corners, int align_mode)
//       -> (Tensor[], Tensor)   (grad_levels, grad_gate)
//   affinity_atrous_pool2d(Tensor feat, Tensor gate, int[] dilations) -> Tensor
//       (CSPN's atrous spatial pyramid pooling: feat (B, C, H, W) and gate (B, 9L, H, W) -> (B, L*C, H, W), level l a 3x3
//       CSPN step dilated by dilations[l])
//   affinity_atrous_pool2d_backward(Tensor feat, Tensor gate, Tensor out, Tensor grad_out, int[] dilations)
//       -> (Tensor, Tensor)   (grad_feat, grad_gate)
// There is no CPU kernel: CPU tensors reach the dispatcher's "no kernel for backend CPU" error, loudly.
#include <ATen/ATen.h>
#include <c10/cuda/CUDAGuard.h>
#include <c10/cuda/CUDAStream.h>
#include <torch/library.h>

#include <algorithm>
#include <optional>
#include <tuple>
#include <utility>
#include <vector>

#include "../../include/cspn_b200.h"

namespace {

// null for an undefined tensor: an absent sparse_depth, a gradient that is not wanted
const float* fptr(const at::Tensor& t) { return t.defined() ? t.data_ptr<float>() : nullptr; }
float* mptr(const at::Tensor& t) { return t.defined() ? t.data_ptr<float>() : nullptr; }

void check_rc(int rc, const char* what) {
    if (rc == CSPN_OK) return;
    const char* msg = cspn_last_error();
    TORCH_CHECK(rc != CSPN_ERR_INVALID_ARGUMENT, what, ": ", msg);
    TORCH_CHECK(false, what, " failed (status ", rc, "): ", msg);
}

// The byte workspace a C ABI call asks for, on the device of `like`; no tensor and a null pointer when it asks for none
struct Workspace {
    size_t bytes;
    at::Tensor t;
    Workspace(size_t bytes, const at::Tensor& like) : bytes(bytes) {
        if (bytes) t = at::empty({(int64_t)bytes}, like.options().dtype(at::kByte));
    }
    void* ptr() const { return bytes ? t.data_ptr() : nullptr; }
};

cspn_stream_t current_stream() { return (cspn_stream_t)c10::cuda::getCurrentCUDAStream().stream(); }

void check_grad_out(const at::Tensor& grad_out, const at::Tensor& x, const char* name) {
    TORCH_CHECK(grad_out.sizes() == x.sizes() && grad_out.scalar_type() == at::kFloat && grad_out.device() == x.device(),
                "grad_out must match ", name);
}

// The gradient of x: allocated when wanted, undefined otherwise.  An unused gradient is returned as an empty tensor (the
// Python autograd formula maps it to None).
at::Tensor new_grad(bool need, const at::Tensor& x) { return need ? at::empty_like(x) : at::Tensor(); }
at::Tensor grad_or_empty(const at::Tensor& grad, const at::Tensor& x) { return grad.defined() ? grad : at::zeros({0}, x.options()); }

// Neighbours of a kernel of size K in nd dimensions, and the sizes the kernels exist for
int64_t neighbours(int64_t K, int nd) { return (nd == 2 ? K * K : K * K * K) - 1; }
bool kernel_size_ok(int64_t K, int nd) { return K == 3 || K == 5 || (nd == 2 && K == 7); }

void check2d(const at::Tensor& guidance, const at::Tensor& blur, const std::optional<at::Tensor>& sparse) {
    TORCH_CHECK(guidance.dim() == 4 && blur.dim() == 4, "guidance and blur_depth must be (B,C,H,W)");
    // the reference raises here too: its ones-weight conv is fp32 (cspn.py:44-53)
    TORCH_CHECK(guidance.scalar_type() == at::kFloat && blur.scalar_type() == at::kFloat, "cspn_b200 is fp32 only");
    TORCH_CHECK(guidance.size(0) == blur.size(0) && guidance.size(2) == blur.size(2) && guidance.size(3) == blur.size(3) &&
                    guidance.size(1) >= 8,
                "guidance ", guidance.sizes(), " does not match blur_depth ", blur.sizes(), " (need (B,>=8,H,W))");
    TORCH_CHECK(guidance.device() == blur.device(), "guidance and blur_depth are on different devices");
    if (sparse.has_value()) {
        TORCH_CHECK(sparse->dim() == 4 && sparse->size(0) == blur.size(0) && sparse->size(1) == 1 &&
                        sparse->size(2) == blur.size(2) && sparse->size(3) == blur.size(3),
                    "sparse_depth must be (B,1,H,W), got ", sparse->sizes());
        TORCH_CHECK(sparse->scalar_type() == at::kFloat && sparse->device() == blur.device(),
                    "sparse_depth must be fp32 on the device of blur_depth");
    }
}

at::Tensor propagate2d_cuda(const at::Tensor& guidance, const at::Tensor& blur, const std::optional<at::Tensor>& sparse,
                            int64_t prop_time, int64_t norm_type, int64_t algo) {
    check2d(guidance, blur, sparse);
    if (prop_time == 0) return blur.clone();           // a dispatcher op may not return its input (cspn.py:61,83 does)
    const c10::cuda::CUDAGuard guard(blur.device());
    const at::Tensor g = guidance.contiguous(), d = blur.contiguous();
    const at::Tensor s = sparse.has_value() ? sparse->contiguous() : at::Tensor();
    at::Tensor out = at::empty_like(d);
    const int B = (int)d.size(0), C = (int)d.size(1), H = (int)d.size(2), W = (int)d.size(3);
    int a = (int)algo;
    auto misaligned = [](const at::Tensor& t) { return t.defined() && (reinterpret_cast<uintptr_t>(t.data_ptr()) & 15) != 0; };
    if (a == CSPN_ALGO_AUTO && (misaligned(g) || misaligned(d) || misaligned(s) || misaligned(out))) a = CSPN_ALGO_GENERIC;
    const Workspace ws(cspn2d_workspace_bytes(B, C, H, W, (int)prop_time, a), d);
    check_rc(cspn2d_fwd_f32(fptr(g), fptr(d), fptr(s), mptr(out), B, C, H, W, (int)g.size(1), (int)prop_time, (int)norm_type, a,
                            ws.ptr(), ws.bytes, current_stream()),
             "cspn2d_fwd_f32");
    return out;
}

std::tuple<at::Tensor, at::Tensor> propagate2d_backward_cuda(const at::Tensor& guidance, const at::Tensor& blur,
                                                             const std::optional<at::Tensor>& sparse, const at::Tensor& grad_out,
                                                             int64_t prop_time, int64_t norm_type, bool need_g, bool need_d) {
    check2d(guidance, blur, sparse);
    check_grad_out(grad_out, blur, "blur_depth");
    const c10::cuda::CUDAGuard guard(blur.device());
    const at::Tensor g = guidance.contiguous(), d = blur.contiguous(), go = grad_out.contiguous();
    const at::Tensor s = sparse.has_value() ? sparse->contiguous() : at::Tensor();
    at::Tensor gg = new_grad(need_g, g), gd = new_grad(need_d, d);
    if (prop_time == 0) {                              // identity: d out / d blur = 1, no dependence on the guidance
        if (need_g) gg.zero_();
        if (need_d) gd.copy_(go);
        return {grad_or_empty(gg, g), grad_or_empty(gd, d)};
    }
    const int B = (int)d.size(0), C = (int)d.size(1), H = (int)d.size(2), W = (int)d.size(3);
    const Workspace ws(cspn2d_bwd_workspace_bytes(B, C, H, W, (int)prop_time), d);
    check_rc(cspn2d_bwd_f32(fptr(g), fptr(d), fptr(s), fptr(go), mptr(gg), mptr(gd), B, C, H, W, (int)g.size(1), (int)prop_time,
                            (int)norm_type, ws.ptr(), ws.bytes, current_stream()),
             "cspn2d_bwd_f32");
    return {grad_or_empty(gg, g), grad_or_empty(gd, d)};
}

// K x K kernels: K = 3 is the 3x3 operator above (same kernels, same bits); K = 5 / 7 go through cspn2d_k_*_f32
void check2d_k(const at::Tensor& guidance, const at::Tensor& blur, const std::optional<at::Tensor>& sparse, int64_t K) {
    TORCH_CHECK(kernel_size_ok(K, 2), "kernel_size must be 3, 5 or 7, got ", K);
    check2d(guidance, blur, sparse);
    TORCH_CHECK(guidance.size(1) >= neighbours(K, 2), "a ", K, "x", K, " kernel needs guidance (B,>=", neighbours(K, 2),
                ",H,W), got ", guidance.sizes());
}

at::Tensor propagate2d_k_cuda(const at::Tensor& guidance, const at::Tensor& blur, const std::optional<at::Tensor>& sparse,
                              int64_t K, int64_t prop_time, int64_t norm_type) {
    check2d_k(guidance, blur, sparse, K);
    if (K == 3) return propagate2d_cuda(guidance, blur, sparse, prop_time, norm_type, CSPN_ALGO_AUTO);
    if (prop_time == 0) return blur.clone();
    const c10::cuda::CUDAGuard guard(blur.device());
    const at::Tensor g = guidance.contiguous(), d = blur.contiguous();
    const at::Tensor s = sparse.has_value() ? sparse->contiguous() : at::Tensor();
    at::Tensor out = at::empty_like(d);
    const int B = (int)d.size(0), C = (int)d.size(1), H = (int)d.size(2), W = (int)d.size(3);
    const Workspace ws(cspn2d_k_workspace_bytes(B, C, H, W, (int)K, (int)prop_time), d);
    check_rc(cspn2d_k_fwd_f32(fptr(g), fptr(d), fptr(s), mptr(out), B, C, H, W, (int)g.size(1), (int)K, (int)prop_time,
                              (int)norm_type, ws.ptr(), ws.bytes, current_stream()),
             "cspn2d_k_fwd_f32");
    return out;
}

std::tuple<at::Tensor, at::Tensor> propagate2d_k_backward_cuda(const at::Tensor& guidance, const at::Tensor& blur,
                                                               const std::optional<at::Tensor>& sparse, const at::Tensor& grad_out,
                                                               int64_t K, int64_t prop_time, int64_t norm_type, bool need_g,
                                                               bool need_d) {
    check2d_k(guidance, blur, sparse, K);
    if (K == 3) return propagate2d_backward_cuda(guidance, blur, sparse, grad_out, prop_time, norm_type, need_g, need_d);
    check_grad_out(grad_out, blur, "blur_depth");
    const c10::cuda::CUDAGuard guard(blur.device());
    const at::Tensor g = guidance.contiguous(), d = blur.contiguous(), go = grad_out.contiguous();
    const at::Tensor s = sparse.has_value() ? sparse->contiguous() : at::Tensor();
    at::Tensor gg = new_grad(need_g, g), gd = new_grad(need_d, d);
    const int B = (int)d.size(0), C = (int)d.size(1), H = (int)d.size(2), W = (int)d.size(3);
    const Workspace ws(cspn2d_k_bwd_workspace_bytes(B, C, H, W, (int)K, (int)prop_time), d);
    check_rc(cspn2d_k_bwd_f32(fptr(g), fptr(d), fptr(s), fptr(go), mptr(gg), mptr(gd), B, C, H, W, (int)g.size(1), (int)K,
                              (int)prop_time, (int)norm_type, ws.ptr(), ws.bytes, current_stream()),
             "cspn2d_k_bwd_f32");
    return {grad_or_empty(gg, g), grad_or_empty(gd, d)};
}

// Keep-sparse mode, K in {3, 5, 7}: cspn2d_keep_*_f32.  algo picks the 3x3 path as in propagate2d (misaligned views take the
// generic one under AUTO); a missing sparse_depth is the default mode
at::Tensor propagate2d_keep_cuda(const at::Tensor& guidance, const at::Tensor& blur, const std::optional<at::Tensor>& sparse,
                                 int64_t K, int64_t prop_time, int64_t norm_type, int64_t algo) {
    check2d_k(guidance, blur, sparse, K);
    if (prop_time == 0) return blur.clone();
    const c10::cuda::CUDAGuard guard(blur.device());
    const at::Tensor g = guidance.contiguous(), d = blur.contiguous();
    const at::Tensor s = sparse.has_value() ? sparse->contiguous() : at::Tensor();
    at::Tensor out = at::empty_like(d);
    const int B = (int)d.size(0), C = (int)d.size(1), H = (int)d.size(2), W = (int)d.size(3);
    int a = (int)algo;
    auto misaligned = [](const at::Tensor& t) { return t.defined() && (reinterpret_cast<uintptr_t>(t.data_ptr()) & 15) != 0; };
    if (a == CSPN_ALGO_AUTO && (misaligned(g) || misaligned(d) || misaligned(s) || misaligned(out))) a = CSPN_ALGO_GENERIC;
    const Workspace ws(cspn2d_keep_workspace_bytes(B, C, H, W, (int)K, (int)prop_time, a), d);
    check_rc(cspn2d_keep_fwd_f32(fptr(g), fptr(d), fptr(s), mptr(out), B, C, H, W, (int)g.size(1), (int)K, (int)prop_time,
                                 (int)norm_type, a, ws.ptr(), ws.bytes, current_stream()),
             "cspn2d_keep_fwd_f32");
    return out;
}

std::tuple<at::Tensor, at::Tensor, at::Tensor> propagate2d_keep_backward_cuda(
        const at::Tensor& guidance, const at::Tensor& blur, const std::optional<at::Tensor>& sparse, const at::Tensor& grad_out,
        int64_t K, int64_t prop_time, int64_t norm_type, bool need_g, bool need_d, bool need_s) {
    check2d_k(guidance, blur, sparse, K);
    check_grad_out(grad_out, blur, "blur_depth");
    const c10::cuda::CUDAGuard guard(blur.device());
    const at::Tensor g = guidance.contiguous(), d = blur.contiguous(), go = grad_out.contiguous();
    const at::Tensor s = sparse.has_value() ? sparse->contiguous() : at::Tensor();
    at::Tensor gg = new_grad(need_g, g), gd = new_grad(need_d, d), gs = s.defined() ? new_grad(need_s, s) : at::Tensor();
    const int B = (int)d.size(0), C = (int)d.size(1), H = (int)d.size(2), W = (int)d.size(3);
    const Workspace ws(cspn2d_keep_bwd_workspace_bytes(B, C, H, W, (int)K, (int)prop_time), d);
    check_rc(cspn2d_keep_bwd_f32(fptr(g), fptr(d), fptr(s), fptr(go), mptr(gg), mptr(gd), mptr(gs), B, C, H, W, (int)g.size(1),
                                 (int)K, (int)prop_time, (int)norm_type, ws.ptr(), ws.bytes, current_stream()),
             "cspn2d_keep_bwd_f32");
    return {grad_or_empty(gg, g), grad_or_empty(gd, d), grad_or_empty(gs, d)};
}

// Aggregation of the steps, K in {3, 5, 7}: cspn2d_agg_*_f32.  step_weight (B, T, H, W) with T = len(steps)
std::vector<int> check2d_agg(const at::Tensor& guidance, const at::Tensor& blur, const std::optional<at::Tensor>& sparse,
                             const at::Tensor& step_weight, at::IntArrayRef steps, int64_t K) {
    check2d_k(guidance, blur, sparse, K);
    TORCH_CHECK(!steps.empty(), "steps must hold at least one step");
    for (size_t j = 0; j < steps.size(); ++j)
        TORCH_CHECK(steps[j] >= 1 && steps[j] <= INT32_MAX && (j == 0 || steps[j] > steps[j - 1]),
                    "steps must be strictly increasing ints >= 1, got ", steps);
    TORCH_CHECK(step_weight.dim() == 4 && step_weight.size(0) == blur.size(0) && step_weight.size(1) == (int64_t)steps.size() &&
                    step_weight.size(2) == blur.size(2) && step_weight.size(3) == blur.size(3),
                "step_weight must be (B, len(steps), H, W), got ", step_weight.sizes());
    TORCH_CHECK(step_weight.scalar_type() == at::kFloat && step_weight.device() == blur.device(),
                "step_weight must be fp32 on the device of blur_depth");
    return std::vector<int>(steps.begin(), steps.end());
}

at::Tensor propagate2d_aggregate_cuda(const at::Tensor& guidance, const at::Tensor& blur, const std::optional<at::Tensor>& sparse,
                                      const at::Tensor& step_weight, at::IntArrayRef steps, int64_t K, int64_t norm_type, bool keep) {
    const std::vector<int> st = check2d_agg(guidance, blur, sparse, step_weight, steps, K);
    const c10::cuda::CUDAGuard guard(blur.device());
    const at::Tensor g = guidance.contiguous(), d = blur.contiguous(), w = step_weight.contiguous();
    const at::Tensor s = sparse.has_value() ? sparse->contiguous() : at::Tensor();
    at::Tensor out = at::empty_like(d);
    const int B = (int)d.size(0), C = (int)d.size(1), H = (int)d.size(2), W = (int)d.size(3), T = (int)st.size();
    const Workspace ws(cspn2d_agg_workspace_bytes(B, C, H, W, (int)K, st.data(), T, keep), d);
    check_rc(cspn2d_agg_fwd_f32(fptr(g), fptr(d), fptr(s), fptr(w), mptr(out), B, C, H, W, (int)g.size(1), (int)K, st.data(), T,
                                (int)norm_type, keep, ws.ptr(), ws.bytes, current_stream()),
             "cspn2d_agg_fwd_f32");
    return out;
}

std::tuple<at::Tensor, at::Tensor, at::Tensor, at::Tensor> propagate2d_aggregate_backward_cuda(
        const at::Tensor& guidance, const at::Tensor& blur, const std::optional<at::Tensor>& sparse, const at::Tensor& step_weight,
        const at::Tensor& grad_out, at::IntArrayRef steps, int64_t K, int64_t norm_type, bool keep, bool need_g, bool need_d,
        bool need_s, bool need_w) {
    const std::vector<int> st = check2d_agg(guidance, blur, sparse, step_weight, steps, K);
    check_grad_out(grad_out, blur, "blur_depth");
    const c10::cuda::CUDAGuard guard(blur.device());
    const at::Tensor g = guidance.contiguous(), d = blur.contiguous(), w = step_weight.contiguous(), go = grad_out.contiguous();
    const at::Tensor s = sparse.has_value() ? sparse->contiguous() : at::Tensor();
    at::Tensor gg = new_grad(need_g, g), gd = new_grad(need_d, d), gs = s.defined() ? new_grad(need_s, s) : at::Tensor(),
               gw = new_grad(need_w, w);
    const int B = (int)d.size(0), C = (int)d.size(1), H = (int)d.size(2), W = (int)d.size(3), T = (int)st.size();
    const Workspace ws(cspn2d_agg_bwd_workspace_bytes(B, C, H, W, (int)K, st.data(), T, keep), d);
    check_rc(cspn2d_agg_bwd_f32(fptr(g), fptr(d), fptr(s), fptr(w), fptr(go), mptr(gg), mptr(gd), mptr(gs), mptr(gw), B, C, H, W,
                                (int)g.size(1), (int)K, st.data(), T, (int)norm_type, keep, ws.ptr(), ws.bytes, current_stream()),
             "cspn2d_agg_bwd_f32");
    return {grad_or_empty(gg, g), grad_or_empty(gd, d), grad_or_empty(gs, d), grad_or_empty(gw, w)};
}

// Non-local propagation, K in {3, 5, 7}: cspn2d_nl_*_f32.  feat (B, C, H, W), offset (B, 2T, H, W), affinity (B, T, H, W),
// sparse_depth of feat's shape
void check2d_nl(const at::Tensor& feat, const at::Tensor& offset, const at::Tensor& affinity, const std::optional<at::Tensor>& sparse,
                int64_t K, int64_t prop_time) {
    TORCH_CHECK_VALUE(kernel_size_ok(K, 2), "kernel_size must be 3, 5 or 7, got ", K);
    TORCH_CHECK_VALUE(prop_time >= 0 && prop_time <= INT32_MAX, "prop_time must be >= 0, got ", prop_time);
    const int64_t T = neighbours(K, 2);
    TORCH_CHECK_VALUE(feat.dim() == 4 && feat.numel() > 0, "feat must be a non-empty (B,C,H,W), got ", feat.sizes());
    const int64_t B = feat.size(0), H = feat.size(2), W = feat.size(3);
    TORCH_CHECK_VALUE(offset.dim() == 4 && offset.size(0) == B && offset.size(1) == 2 * T && offset.size(2) == H && offset.size(3) == W,
                      "offset must be (B, 2T, H, W) = (", B, ", ", 2 * T, ", ", H, ", ", W, "), got ", offset.sizes());
    TORCH_CHECK_VALUE(affinity.dim() == 4 && affinity.size(0) == B && affinity.size(1) == T && affinity.size(2) == H &&
                          affinity.size(3) == W,
                      "affinity must be (B, T, H, W) = (", B, ", ", T, ", ", H, ", ", W, "), got ", affinity.sizes());
    TORCH_CHECK(feat.scalar_type() == at::kFloat && offset.scalar_type() == at::kFloat && affinity.scalar_type() == at::kFloat,
                "cspn_b200 is fp32 only");
    TORCH_CHECK(offset.device() == feat.device() && affinity.device() == feat.device(), "feat, offset and affinity are on different devices");
    if (sparse.has_value()) {
        TORCH_CHECK_VALUE(sparse->sizes() == feat.sizes(), "sparse_depth must have feat's shape ", feat.sizes(), ", got ", sparse->sizes());
        TORCH_CHECK(sparse->scalar_type() == at::kFloat && sparse->device() == feat.device(), "sparse_depth must be fp32 on the device of feat");
    }
    TORCH_CHECK(B < ((int64_t)1 << 31) && feat.size(1) < ((int64_t)1 << 31) && H * W * T < ((int64_t)1 << 31),
                "propagate2d_nonlocal takes B, C < 2^31 and H*W*T < 2^31, got feat ", feat.sizes(), " at K=", K);
}

at::Tensor propagate2d_nonlocal_cuda(const at::Tensor& feat, const at::Tensor& offset, const at::Tensor& affinity,
                                     const std::optional<at::Tensor>& sparse, int64_t K, int64_t prop_time) {
    check2d_nl(feat, offset, affinity, sparse, K, prop_time);
    if (prop_time == 0) return feat.clone();           // a dispatcher op may not return its input
    const c10::cuda::CUDAGuard guard(feat.device());
    const at::Tensor f = feat.contiguous(), o = offset.contiguous(), a = affinity.contiguous();
    const at::Tensor s = sparse.has_value() ? sparse->contiguous() : at::Tensor();
    at::Tensor out = at::empty_like(f);
    const int B = (int)f.size(0), C = (int)f.size(1), H = (int)f.size(2), W = (int)f.size(3);
    const Workspace ws(cspn2d_nl_workspace_bytes(B, C, H, W, (int)K, (int)prop_time), f);
    check_rc(cspn2d_nl_fwd_f32(fptr(f), fptr(o), fptr(a), fptr(s), mptr(out), B, C, H, W, (int)K, (int)prop_time, ws.ptr(), ws.bytes,
                               current_stream()),
             "cspn2d_nl_fwd_f32");
    return out;
}

std::tuple<at::Tensor, at::Tensor, at::Tensor, at::Tensor> propagate2d_nonlocal_backward_cuda(
        const at::Tensor& feat, const at::Tensor& offset, const at::Tensor& affinity, const std::optional<at::Tensor>& sparse,
        const at::Tensor& grad_out, int64_t K, int64_t prop_time, bool need_f, bool need_o, bool need_a, bool need_s) {
    check2d_nl(feat, offset, affinity, sparse, K, prop_time);
    check_grad_out(grad_out, feat, "feat");
    const c10::cuda::CUDAGuard guard(feat.device());
    const at::Tensor f = feat.contiguous(), o = offset.contiguous(), a = affinity.contiguous(), go = grad_out.contiguous();
    const at::Tensor s = sparse.has_value() ? sparse->contiguous() : at::Tensor();
    at::Tensor gf = new_grad(need_f, f), gof = new_grad(need_o, o), ga = new_grad(need_a, a),
               gs = s.defined() ? new_grad(need_s, s) : at::Tensor();
    const int B = (int)f.size(0), C = (int)f.size(1), H = (int)f.size(2), W = (int)f.size(3);
    const Workspace ws(prop_time > 0 ? cspn2d_nl_bwd_workspace_bytes(B, C, H, W, (int)K, (int)prop_time) : 0, f);
    check_rc(cspn2d_nl_bwd_f32(fptr(f), fptr(o), fptr(a), fptr(s), fptr(go), mptr(gf), mptr(gof), mptr(ga), mptr(gs), B, C, H, W, (int)K,
                               (int)prop_time, ws.ptr(), ws.bytes, current_stream()),
             "cspn2d_nl_bwd_f32");
    return {grad_or_empty(gf, f), grad_or_empty(gof, o), grad_or_empty(ga, a), grad_or_empty(gs, f)};
}

// Dilated propagation, K in {3, 5, 7}: cspn2d_dil_*_f32.  kernel (B, K*K, H, W), blur_depth (B, C, H, W), sparse_depth and
// confidence (B, 1, H, W), both or neither
void check2d_dil(const at::Tensor& kernel, const at::Tensor& blur, const std::optional<at::Tensor>& sparse,
                 const std::optional<at::Tensor>& conf, int64_t K, int64_t dilation, int64_t prop_time) {
    TORCH_CHECK_VALUE(kernel_size_ok(K, 2), "kernel_size must be 3, 5 or 7, got ", K);
    TORCH_CHECK_VALUE(dilation >= 1 && dilation <= 4, "dilation must be in [1, 4], got ", dilation);
    TORCH_CHECK_VALUE(prop_time >= 0 && prop_time <= INT32_MAX, "prop_time must be >= 0, got ", prop_time);
    TORCH_CHECK_VALUE(sparse.has_value() == conf.has_value(), "sparse_depth and confidence come together or not at all");
    TORCH_CHECK_VALUE(blur.dim() == 4 && blur.numel() > 0, "blur_depth must be a non-empty (B,C,H,W), got ", blur.sizes());
    const int64_t B = blur.size(0), C = blur.size(1), H = blur.size(2), W = blur.size(3);
    TORCH_CHECK_VALUE(kernel.dim() == 4 && kernel.size(0) == B && kernel.size(1) == K * K && kernel.size(2) == H && kernel.size(3) == W,
                      "kernel must be (B, K*K, H, W) = (", B, ", ", K * K, ", ", H, ", ", W, "), got ", kernel.sizes());
    TORCH_CHECK(kernel.scalar_type() == at::kFloat && blur.scalar_type() == at::kFloat, "cspn_b200 is fp32 only");
    TORCH_CHECK(kernel.device() == blur.device(), "kernel and blur_depth are on different devices");
    for (const auto* t : {&sparse, &conf})
        if (t->has_value()) {
            TORCH_CHECK_VALUE((*t)->dim() == 4 && (*t)->size(0) == B && (*t)->size(1) == 1 && (*t)->size(2) == H && (*t)->size(3) == W,
                              "sparse_depth and confidence must be (B, 1, H, W) = (", B, ", 1, ", H, ", ", W, "), got ", (*t)->sizes());
            TORCH_CHECK((*t)->scalar_type() == at::kFloat && (*t)->device() == blur.device(),
                        "sparse_depth and confidence must be fp32 on the device of blur_depth");
        }
    TORCH_CHECK(B * C <= 65535 && (H + 15) / 16 <= 65535 && W < ((int64_t)1 << 31),
                "propagate2d_dilated takes B*C <= 65535 and ceil(H/16) <= 65535, got blur_depth ", blur.sizes());
}

at::Tensor propagate2d_dilated_cuda(const at::Tensor& kernel, const at::Tensor& blur, const std::optional<at::Tensor>& sparse,
                                    const std::optional<at::Tensor>& conf, int64_t K, int64_t dilation, int64_t prop_time) {
    check2d_dil(kernel, blur, sparse, conf, K, dilation, prop_time);
    if (prop_time == 0) return blur.clone();           // a dispatcher op may not return its input
    const c10::cuda::CUDAGuard guard(blur.device());
    const at::Tensor k = kernel.contiguous(), d = blur.contiguous();
    const at::Tensor s = sparse.has_value() ? sparse->contiguous() : at::Tensor();
    const at::Tensor m = conf.has_value() ? conf->contiguous() : at::Tensor();
    at::Tensor out = at::empty_like(d);
    const int B = (int)d.size(0), C = (int)d.size(1), H = (int)d.size(2), W = (int)d.size(3);
    const Workspace ws(cspn2d_dil_workspace_bytes(B, C, H, W, (int)K, (int)dilation, (int)prop_time), d);
    check_rc(cspn2d_dil_fwd_f32(fptr(k), fptr(d), fptr(s), fptr(m), mptr(out), B, C, H, W, (int)K, (int)dilation, (int)prop_time,
                                ws.ptr(), ws.bytes, current_stream()),
             "cspn2d_dil_fwd_f32");
    return out;
}

std::tuple<at::Tensor, at::Tensor, at::Tensor, at::Tensor> propagate2d_dilated_backward_cuda(
        const at::Tensor& kernel, const at::Tensor& blur, const std::optional<at::Tensor>& sparse, const std::optional<at::Tensor>& conf,
        const at::Tensor& grad_out, int64_t K, int64_t dilation, int64_t prop_time, bool need_k, bool need_d, bool need_s, bool need_m) {
    check2d_dil(kernel, blur, sparse, conf, K, dilation, prop_time);
    check_grad_out(grad_out, blur, "blur_depth");
    const c10::cuda::CUDAGuard guard(blur.device());
    const at::Tensor k = kernel.contiguous(), d = blur.contiguous(), go = grad_out.contiguous();
    const at::Tensor s = sparse.has_value() ? sparse->contiguous() : at::Tensor();
    const at::Tensor m = conf.has_value() ? conf->contiguous() : at::Tensor();
    at::Tensor gk = new_grad(need_k, k), gd = new_grad(need_d, d);
    at::Tensor gs = s.defined() ? new_grad(need_s, s) : at::Tensor(), gm = m.defined() ? new_grad(need_m, m) : at::Tensor();
    const int B = (int)d.size(0), C = (int)d.size(1), H = (int)d.size(2), W = (int)d.size(3);
    const Workspace ws(cspn2d_dil_bwd_workspace_bytes(B, C, H, W, (int)K, (int)dilation, (int)prop_time), d);
    check_rc(cspn2d_dil_bwd_f32(fptr(k), fptr(d), fptr(s), fptr(m), fptr(go), mptr(gk), mptr(gd), mptr(gs), mptr(gm), B, C, H, W, (int)K,
                                (int)dilation, (int)prop_time, ws.ptr(), ws.bytes, current_stream()),
             "cspn2d_dil_bwd_f32");
    return {grad_or_empty(gk, k), grad_or_empty(gd, d), grad_or_empty(gs, d), grad_or_empty(gm, d)};
}

// Dynamic propagation, K in {3, 5, 7}: cspn2d_dyn_*_f32.  affinity (B, K*K, H, W), attention (B, N*(K+1)/2, H, W), blur_depth
// (B, C, H, W), sparse_depth and confidence (B, 1, H, W), both or neither.  Returns N.
int64_t check2d_dyn(const at::Tensor& aff, const at::Tensor& att, const at::Tensor& blur, const std::optional<at::Tensor>& sparse,
                    const std::optional<at::Tensor>& conf, int64_t K) {
    TORCH_CHECK_VALUE(kernel_size_ok(K, 2), "kernel_size must be 3, 5 or 7, got ", K);
    TORCH_CHECK_VALUE(sparse.has_value() == conf.has_value(), "sparse_depth and confidence come together or not at all");
    TORCH_CHECK_VALUE(blur.dim() == 4 && blur.numel() > 0, "blur_depth must be a non-empty (B,C,H,W), got ", blur.sizes());
    const int64_t B = blur.size(0), C = blur.size(1), H = blur.size(2), W = blur.size(3), NR = (K + 1) / 2;
    TORCH_CHECK_VALUE(aff.dim() == 4 && aff.size(0) == B && aff.size(1) == K * K && aff.size(2) == H && aff.size(3) == W,
                      "affinity must be (B, K*K, H, W) = (", B, ", ", K * K, ", ", H, ", ", W, "), got ", aff.sizes());
    TORCH_CHECK_VALUE(att.dim() == 4 && att.size(0) == B && att.size(1) % NR == 0 && att.size(2) == H && att.size(3) == W &&
                              att.size(1) <= INT32_MAX,
                      "attention must be (B, N*(K+1)/2, H, W) with (K+1)/2 = ", NR, " and H, W = ", H, ", ", W, ", got ", att.sizes());
    TORCH_CHECK(aff.scalar_type() == at::kFloat && att.scalar_type() == at::kFloat && blur.scalar_type() == at::kFloat,
                "cspn_b200 is fp32 only");
    TORCH_CHECK(aff.device() == blur.device() && att.device() == blur.device(), "affinity, attention and blur_depth are on different devices");
    for (const auto* t : {&sparse, &conf})
        if (t->has_value()) {
            TORCH_CHECK_VALUE((*t)->dim() == 4 && (*t)->size(0) == B && (*t)->size(1) == 1 && (*t)->size(2) == H && (*t)->size(3) == W,
                              "sparse_depth and confidence must be (B, 1, H, W) = (", B, ", 1, ", H, ", ", W, "), got ", (*t)->sizes());
            TORCH_CHECK((*t)->scalar_type() == at::kFloat && (*t)->device() == blur.device(),
                        "sparse_depth and confidence must be fp32 on the device of blur_depth");
        }
    TORCH_CHECK(B * C <= 65535 && (H + 15) / 16 <= 65535 && W < ((int64_t)1 << 31),
                "propagate2d_dynamic takes B*C <= 65535 and ceil(H/16) <= 65535, got blur_depth ", blur.sizes());
    return att.size(1) / NR;
}

at::Tensor propagate2d_dynamic_cuda(const at::Tensor& aff, const at::Tensor& att, const at::Tensor& blur,
                                    const std::optional<at::Tensor>& sparse, const std::optional<at::Tensor>& conf, int64_t K) {
    const int64_t N = check2d_dyn(aff, att, blur, sparse, conf, K);
    if (N == 0) return blur.clone();                   // a dispatcher op may not return its input
    const c10::cuda::CUDAGuard guard(blur.device());
    const at::Tensor a = aff.contiguous(), at_ = att.contiguous(), d = blur.contiguous();
    const at::Tensor s = sparse.has_value() ? sparse->contiguous() : at::Tensor();
    const at::Tensor m = conf.has_value() ? conf->contiguous() : at::Tensor();
    at::Tensor out = at::empty_like(d);
    const int B = (int)d.size(0), C = (int)d.size(1), H = (int)d.size(2), W = (int)d.size(3);
    const Workspace ws(cspn2d_dyn_workspace_bytes(B, C, H, W, (int)K, (int)N), d);
    check_rc(cspn2d_dyn_fwd_f32(fptr(a), fptr(at_), fptr(d), fptr(s), fptr(m), mptr(out), B, C, H, W, (int)K, (int)N, ws.ptr(), ws.bytes,
                                current_stream()),
             "cspn2d_dyn_fwd_f32");
    return out;
}

std::tuple<at::Tensor, at::Tensor, at::Tensor, at::Tensor, at::Tensor> propagate2d_dynamic_backward_cuda(
        const at::Tensor& aff, const at::Tensor& att, const at::Tensor& blur, const std::optional<at::Tensor>& sparse,
        const std::optional<at::Tensor>& conf, const at::Tensor& grad_out, int64_t K, bool need_a, bool need_att, bool need_d, bool need_s,
        bool need_m) {
    const int64_t N = check2d_dyn(aff, att, blur, sparse, conf, K);
    check_grad_out(grad_out, blur, "blur_depth");
    const c10::cuda::CUDAGuard guard(blur.device());
    const at::Tensor a = aff.contiguous(), at_ = att.contiguous(), d = blur.contiguous(), go = grad_out.contiguous();
    const at::Tensor s = sparse.has_value() ? sparse->contiguous() : at::Tensor();
    const at::Tensor m = conf.has_value() ? conf->contiguous() : at::Tensor();
    at::Tensor ga = new_grad(need_a, a), gt = new_grad(need_att, at_), gd = new_grad(need_d, d);
    at::Tensor gs = s.defined() ? new_grad(need_s, s) : at::Tensor(), gm = m.defined() ? new_grad(need_m, m) : at::Tensor();
    const int B = (int)d.size(0), C = (int)d.size(1), H = (int)d.size(2), W = (int)d.size(3);
    const Workspace ws(cspn2d_dyn_bwd_workspace_bytes(B, C, H, W, (int)K, (int)N), d);
    check_rc(cspn2d_dyn_bwd_f32(fptr(a), fptr(at_), fptr(d), fptr(s), fptr(m), fptr(go), mptr(ga), mptr(gt), mptr(gd), mptr(gs), mptr(gm), B,
                                C, H, W, (int)K, (int)N, ws.ptr(), ws.bytes, current_stream()),
             "cspn2d_dyn_bwd_f32");
    return {grad_or_empty(ga, a), grad_or_empty(gt, at_), grad_or_empty(gd, d), grad_or_empty(gs, d), grad_or_empty(gm, d)};
}

// Linear three-way scans (SPN): cspn2d_lin_*_f32.  feat (B, C, H, W), gate (B, 3*nd, H, W) or (B, 3*nd*C, H, W) with C > 1.
// Returns the gate mode.
int check2d_lin(const at::Tensor& feat, const at::Tensor& gate, int64_t mask) {
    TORCH_CHECK_VALUE(mask >= 1 && mask <= 15, "dir_mask must be 1 .. 15, got ", mask);
    TORCH_CHECK_VALUE(feat.dim() == 4 && feat.numel() > 0, "feat must be a non-empty (B,C,H,W), got ", feat.sizes());
    const int64_t B = feat.size(0), C = feat.size(1), H = feat.size(2), W = feat.size(3), nd = __builtin_popcountll(mask);
    TORCH_CHECK_VALUE(gate.dim() == 4 && gate.size(0) == B && gate.size(2) == H && gate.size(3) == W &&
                              (gate.size(1) == 3 * nd || (C > 1 && gate.size(1) == 3 * nd * C)),
                      "gate must be (B, 3*nd, H, W) or, with C > 1, (B, 3*nd*C, H, W), nd = ", nd, ", feat ", feat.sizes(), ", got ",
                      gate.sizes());
    TORCH_CHECK(feat.scalar_type() == at::kFloat && gate.scalar_type() == at::kFloat, "cspn_b200 is fp32 only");
    TORCH_CHECK(gate.device() == feat.device(), "feat and gate are on different devices");
    const int64_t lat = std::max<int64_t>((mask & 3) ? H : 0, (mask & 12) ? W : 0);
    TORCH_CHECK(B * C <= INT32_MAX && lat <= 2048 && gate.size(1) <= INT32_MAX && H * W <= INT32_MAX,
                "propagate2d_linear takes B*C <= 2^31 - 1 and a lateral extent (H for l2r / r2l, W for t2b / b2t) <= 2048, got feat ",
                feat.sizes());
    return gate.size(1) == 3 * nd ? CSPN_LIN_GATE_SHARED : CSPN_LIN_GATE_PER_CHANNEL;
}

std::tuple<at::Tensor, at::Tensor> propagate2d_linear_cuda(const at::Tensor& feat, const at::Tensor& gate, int64_t mask) {
    const int mode = check2d_lin(feat, gate, mask);
    const c10::cuda::CUDAGuard guard(feat.device());
    const at::Tensor x = feat.contiguous(), g = gate.contiguous();
    const int B = (int)x.size(0), C = (int)x.size(1), H = (int)x.size(2), W = (int)x.size(3), nd = __builtin_popcount((int)mask);
    at::Tensor out = at::empty_like(x);
    at::Tensor planes = nd > 1 ? at::empty({nd, B, C, H, W}, x.options()) : at::zeros({0}, x.options());
    check_rc(cspn2d_lin_fwd_f32(fptr(x), fptr(g), mptr(out), nd > 1 ? mptr(planes) : nullptr, B, C, H, W, (int)mask, mode, nullptr, 0,
                                current_stream()),
             "cspn2d_lin_fwd_f32");
    return {out, planes};
}

std::tuple<at::Tensor, at::Tensor> propagate2d_linear_backward_cuda(const at::Tensor& feat, const at::Tensor& gate, const at::Tensor& planes,
                                                                    const at::Tensor& grad_out, int64_t mask, bool need_x, bool need_g) {
    const int mode = check2d_lin(feat, gate, mask);
    check_grad_out(grad_out, feat, "feat");
    const int64_t nd = __builtin_popcountll(mask);
    TORCH_CHECK_VALUE(planes.numel() == nd * feat.numel() && planes.scalar_type() == at::kFloat && planes.device() == feat.device(),
                      "planes must hold the forward's nd = ", nd, " planes of feat's shape, got ", planes.sizes());
    const c10::cuda::CUDAGuard guard(feat.device());
    const at::Tensor x = feat.contiguous(), g = gate.contiguous(), p = planes.contiguous(), go = grad_out.contiguous();
    at::Tensor gx = new_grad(need_x, x), gg = new_grad(need_g, g);
    const int B = (int)x.size(0), C = (int)x.size(1), H = (int)x.size(2), W = (int)x.size(3);
    const Workspace ws(cspn2d_lin_bwd_workspace_bytes(B, C, H, W, (int)mask, mode), x);
    check_rc(cspn2d_lin_bwd_f32(fptr(x), fptr(g), fptr(p), fptr(go), mptr(gx), mptr(gg), B, C, H, W, (int)mask, mode, ws.ptr(), ws.bytes,
                                current_stream()),
             "cspn2d_lin_bwd_f32");
    return {grad_or_empty(gx, x), grad_or_empty(gg, g)};
}

// 2D 'paddle' (own-location gates), K in {3, 5, 7}.  guidance (B, K*K-1, H, W) is shared by the C channels of feat;
// (B, (K*K-1)*C, H, W) with C > 1 gives channel c its own gate (demo.py:28-45), which in memory is B*C images of one
// channel.  Returns the (images, channels) the C ABI is called with.
std::pair<int, int> check2d_paddle(const at::Tensor& guidance, const at::Tensor& feat, int64_t K) {
    TORCH_CHECK_VALUE(kernel_size_ok(K, 2), "kernel_size must be 3, 5 or 7, got ", K);
    TORCH_CHECK_VALUE(guidance.dim() == 4 && feat.dim() == 4, "guidance and feat must be (B,C,H,W)");
    TORCH_CHECK(guidance.scalar_type() == at::kFloat && feat.scalar_type() == at::kFloat, "cspn_b200 is fp32 only");
    const int64_t nt = neighbours(K, 2), B = feat.size(0), C = feat.size(1);
    const bool shape_ok = guidance.size(0) == B && guidance.size(2) == feat.size(2) && guidance.size(3) == feat.size(3);
    const bool per_channel = C > 1 && guidance.size(1) == nt * C;
    TORCH_CHECK_VALUE(shape_ok && (guidance.size(1) == nt || per_channel), "a ", K, "x", K, " 'paddle' kernel needs guidance (B,",
                      nt, ",H,W) or, with C > 1 feature channels, (B,", nt, "*C,H,W); got ", guidance.sizes(), " for feat ",
                      feat.sizes());
    TORCH_CHECK(guidance.device() == feat.device(), "guidance and feat are on different devices");
    return per_channel ? std::make_pair((int)(B * C), 1) : std::make_pair((int)B, (int)C);
}

at::Tensor propagate2d_paddle_cuda(const at::Tensor& guidance, const at::Tensor& feat, int64_t K, int64_t prop_time) {
    const auto [B, C] = check2d_paddle(guidance, feat, K);
    if (prop_time == 0) return feat.clone();
    const c10::cuda::CUDAGuard guard(feat.device());
    const at::Tensor g = guidance.contiguous(), f = feat.contiguous();
    at::Tensor out = at::empty_like(f);
    const int H = (int)f.size(2), W = (int)f.size(3);
    const Workspace ws(cspn2d_paddle_workspace_bytes(B, C, H, W, (int)K, (int)prop_time), f);
    check_rc(cspn2d_paddle_fwd_f32(fptr(g), fptr(f), mptr(out), B, C, H, W, (int)K, (int)prop_time, ws.ptr(), ws.bytes,
                                   current_stream()),
             "cspn2d_paddle_fwd_f32");
    return out;
}

std::tuple<at::Tensor, at::Tensor> propagate2d_paddle_backward_cuda(const at::Tensor& guidance, const at::Tensor& feat,
                                                                    const at::Tensor& grad_out, int64_t K, int64_t prop_time,
                                                                    bool need_g, bool need_f) {
    const auto [B, C] = check2d_paddle(guidance, feat, K);
    check_grad_out(grad_out, feat, "feat");
    const c10::cuda::CUDAGuard guard(feat.device());
    const at::Tensor g = guidance.contiguous(), f = feat.contiguous(), go = grad_out.contiguous();
    at::Tensor gg = new_grad(need_g, g), gf = new_grad(need_f, f);
    const int H = (int)f.size(2), W = (int)f.size(3);
    const Workspace ws(cspn2d_paddle_bwd_workspace_bytes(B, C, H, W, (int)K, (int)prop_time), f);
    check_rc(cspn2d_paddle_bwd_f32(fptr(g), fptr(f), fptr(go), mptr(gg), mptr(gf), B, C, H, W, (int)K, (int)prop_time, ws.ptr(),
                                   ws.bytes, current_stream()),
             "cspn2d_paddle_bwd_f32");
    return {grad_or_empty(gg, g), grad_or_empty(gf, f)};
}

void check3d(const at::Tensor& guidance, const at::Tensor& feat) {
    TORCH_CHECK(guidance.dim() == 5 && feat.dim() == 5, "guidance and feat must be (B,C,D,H,W)");
    TORCH_CHECK(guidance.scalar_type() == at::kFloat && feat.scalar_type() == at::kFloat, "cspn_b200 is fp32 only");
    TORCH_CHECK(guidance.size(0) == feat.size(0) && guidance.size(1) == 26 && guidance.size(2) == feat.size(2) &&
                    guidance.size(3) == feat.size(3) && guidance.size(4) == feat.size(4),
                "guidance must be (B,26,D,H,W), got ", guidance.sizes(), " for feat ", feat.sizes());
    TORCH_CHECK(guidance.device() == feat.device(), "guidance and feat are on different devices");
}

at::Tensor propagate3d_cuda(const at::Tensor& guidance, const at::Tensor& feat, int64_t prop_time, int64_t norm_type) {
    check3d(guidance, feat);
    if (prop_time == 0) return feat.clone();
    const c10::cuda::CUDAGuard guard(feat.device());
    const at::Tensor g = guidance.contiguous(), f = feat.contiguous();
    at::Tensor out = at::empty_like(f);
    const int B = (int)f.size(0), C = (int)f.size(1), D = (int)f.size(2), H = (int)f.size(3), W = (int)f.size(4);
    const Workspace ws(cspn3d_workspace_bytes(B, C, D, H, W, (int)prop_time), f);
    check_rc(cspn3d_fwd_f32(fptr(g), fptr(f), mptr(out), B, C, D, H, W, (int)prop_time, (int)norm_type, ws.ptr(), ws.bytes,
                            current_stream()),
             "cspn3d_fwd_f32");
    return out;
}

std::tuple<at::Tensor, at::Tensor> propagate3d_backward_cuda(const at::Tensor& guidance, const at::Tensor& feat,
                                                             const at::Tensor& grad_out, int64_t prop_time, int64_t norm_type,
                                                             bool need_g, bool need_f) {
    check3d(guidance, feat);
    check_grad_out(grad_out, feat, "feat");
    const c10::cuda::CUDAGuard guard(feat.device());
    const at::Tensor g = guidance.contiguous(), f = feat.contiguous(), go = grad_out.contiguous();
    at::Tensor gg = new_grad(need_g, g), gf = new_grad(need_f, f);
    if (prop_time == 0) {
        if (need_g) gg.zero_();
        if (need_f) gf.copy_(go);
        return {grad_or_empty(gg, g), grad_or_empty(gf, f)};
    }
    const int B = (int)f.size(0), C = (int)f.size(1), D = (int)f.size(2), H = (int)f.size(3), W = (int)f.size(4);
    const Workspace ws(cspn3d_bwd_workspace_bytes(B, C, D, H, W, (int)prop_time), f);
    check_rc(cspn3d_bwd_f32(fptr(g), fptr(f), fptr(go), mptr(gg), mptr(gf), B, C, D, H, W, (int)prop_time, (int)norm_type,
                            ws.ptr(), ws.bytes, current_stream()),
             "cspn3d_bwd_f32");
    return {grad_or_empty(gg, g), grad_or_empty(gf, f)};
}

// K x K x K kernels: K = 3 is the 3D operator above (same kernels, same bits); K = 5 goes through cspn3d_k_*_f32
void check3d_k(const at::Tensor& guidance, const at::Tensor& feat, int64_t K) {
    TORCH_CHECK_VALUE(kernel_size_ok(K, 3), "3D kernel_size must be 3 or 5, got ", K);
    TORCH_CHECK_VALUE(guidance.dim() == 5 && feat.dim() == 5, "guidance and feat must be (B,C,D,H,W)");
    TORCH_CHECK(guidance.scalar_type() == at::kFloat && feat.scalar_type() == at::kFloat, "cspn_b200 is fp32 only");
    const int64_t nt = neighbours(K, 3);
    TORCH_CHECK_VALUE(guidance.size(0) == feat.size(0) && guidance.size(1) == nt && guidance.size(2) == feat.size(2) &&
                          guidance.size(3) == feat.size(3) && guidance.size(4) == feat.size(4),
                      "a ", K, "x", K, "x", K, " kernel needs guidance (B,", nt, ",D,H,W), got ", guidance.sizes(), " for feat ",
                      feat.sizes());
    TORCH_CHECK(guidance.device() == feat.device(), "guidance and feat are on different devices");
}

at::Tensor propagate3d_k_cuda(const at::Tensor& guidance, const at::Tensor& feat, int64_t K, int64_t prop_time, int64_t norm_type) {
    check3d_k(guidance, feat, K);
    if (K == 3) return propagate3d_cuda(guidance, feat, prop_time, norm_type);
    if (prop_time == 0) return feat.clone();
    const c10::cuda::CUDAGuard guard(feat.device());
    const at::Tensor g = guidance.contiguous(), f = feat.contiguous();
    at::Tensor out = at::empty_like(f);
    const int B = (int)f.size(0), C = (int)f.size(1), D = (int)f.size(2), H = (int)f.size(3), W = (int)f.size(4);
    const Workspace ws(cspn3d_k_workspace_bytes(B, C, D, H, W, (int)K, (int)prop_time), f);
    check_rc(cspn3d_k_fwd_f32(fptr(g), fptr(f), mptr(out), B, C, D, H, W, (int)K, (int)prop_time, (int)norm_type, ws.ptr(),
                              ws.bytes, current_stream()),
             "cspn3d_k_fwd_f32");
    return out;
}

std::tuple<at::Tensor, at::Tensor> propagate3d_k_backward_cuda(const at::Tensor& guidance, const at::Tensor& feat,
                                                               const at::Tensor& grad_out, int64_t K, int64_t prop_time,
                                                               int64_t norm_type, bool need_g, bool need_f) {
    check3d_k(guidance, feat, K);
    if (K == 3) return propagate3d_backward_cuda(guidance, feat, grad_out, prop_time, norm_type, need_g, need_f);
    check_grad_out(grad_out, feat, "feat");
    const c10::cuda::CUDAGuard guard(feat.device());
    const at::Tensor g = guidance.contiguous(), f = feat.contiguous(), go = grad_out.contiguous();
    at::Tensor gg = new_grad(need_g, g), gf = new_grad(need_f, f);
    const int B = (int)f.size(0), C = (int)f.size(1), D = (int)f.size(2), H = (int)f.size(3), W = (int)f.size(4);
    const Workspace ws(cspn3d_k_bwd_workspace_bytes(B, C, D, H, W, (int)K, (int)prop_time), f);
    check_rc(cspn3d_k_bwd_f32(fptr(g), fptr(f), fptr(go), mptr(gg), mptr(gf), B, C, D, H, W, (int)K, (int)prop_time,
                              (int)norm_type, ws.ptr(), ws.bytes, current_stream()),
             "cspn3d_k_bwd_f32");
    return {grad_or_empty(gg, g), grad_or_empty(gf, f)};
}

// caller-supplied gates (fluid.layers.affinity_propagate), nd = 2 (K in {3, 5, 7}) or 3 (K in {3, 5}).  Returns the
// (images, channels) the C ABI is called with: per-channel gates are B*C images of one channel.
std::pair<int, int> check_gates(const at::Tensor& input, const at::Tensor& gate, int64_t K, int64_t prop_step, int nd) {
    TORCH_CHECK_VALUE(input.dim() == nd + 2 && gate.dim() == nd + 2, "input and gate_weight must be ",
                      nd == 2 ? "(B,C,H,W)" : "(B,C,D,H,W)");
    TORCH_CHECK_VALUE(kernel_size_ok(K, nd), "kernel_size of a ", nd, "D affinity_propagate must be ",
                      nd == 2 ? "3, 5 or 7" : "3 or 5", ", got ", K);
    TORCH_CHECK_VALUE(prop_step >= 0, "prop_step must be >= 0, got ", prop_step);
    TORCH_CHECK(input.scalar_type() == at::kFloat && gate.scalar_type() == at::kFloat, "cspn_b200 is fp32 only");
    const int64_t nt = neighbours(K, nd), B = input.size(0), C = input.size(1);
    bool shape_ok = gate.size(0) == B;
    for (int i = 2; i < nd + 2; ++i) shape_ok = shape_ok && gate.size(i) == input.size(i);
    const bool per_channel = C > 1 && gate.size(1) == nt * C;
    TORCH_CHECK_VALUE(shape_ok && (gate.size(1) == nt || per_channel), "a kernel of size ", K, " needs gate_weight (B,", nt,
                      ",...) or, with C > 1 input channels, (B,", nt, "*C,...); got ", gate.sizes(), " for input ", input.sizes());
    TORCH_CHECK(gate.device() == input.device(), "input and gate_weight are on different devices");
    return per_channel ? std::make_pair((int)(B * C), 1) : std::make_pair((int)B, (int)C);
}

at::Tensor affinity_propagate_cuda(const at::Tensor& input, const at::Tensor& gate, int64_t K, int64_t prop_step, int nd) {
    const auto [B, C] = check_gates(input, gate, K, prop_step, nd);
    if (prop_step == 0) return input.clone();
    const c10::cuda::CUDAGuard guard(input.device());
    const at::Tensor g = gate.contiguous(), x = input.contiguous();
    at::Tensor out = at::empty_like(x);
    const int H = (int)x.size(nd), W = (int)x.size(nd + 1), D = nd == 3 ? (int)x.size(2) : 1;
    const Workspace ws(nd == 2 ? cspn2d_gates_workspace_bytes(B, C, H, W, (int)K, (int)prop_step)
                               : cspn3d_gates_workspace_bytes(B, C, D, H, W, (int)K, (int)prop_step),
                       x);
    if (nd == 2)
        check_rc(cspn2d_gates_fwd_f32(fptr(g), fptr(x), mptr(out), B, C, H, W, (int)K, (int)prop_step, ws.ptr(), ws.bytes,
                                      current_stream()),
                 "cspn2d_gates_fwd_f32");
    else
        check_rc(cspn3d_gates_fwd_f32(fptr(g), fptr(x), mptr(out), B, C, D, H, W, (int)K, (int)prop_step, ws.ptr(), ws.bytes,
                                      current_stream()),
                 "cspn3d_gates_fwd_f32");
    return out;
}

std::tuple<at::Tensor, at::Tensor> affinity_propagate_backward_cuda(const at::Tensor& input, const at::Tensor& gate,
                                                                    const at::Tensor& grad_out, int64_t K, int64_t prop_step,
                                                                    bool need_x, bool need_g, int nd) {
    const auto [B, C] = check_gates(input, gate, K, prop_step, nd);
    check_grad_out(grad_out, input, "input");
    const c10::cuda::CUDAGuard guard(input.device());
    const at::Tensor g = gate.contiguous(), x = input.contiguous(), go = grad_out.contiguous();
    at::Tensor gx = new_grad(need_x, x), gg = new_grad(need_g, g);
    const int H = (int)x.size(nd), W = (int)x.size(nd + 1), D = nd == 3 ? (int)x.size(2) : 1;
    const Workspace ws(nd == 2 ? cspn2d_gates_bwd_workspace_bytes(B, C, H, W, (int)K, (int)prop_step)
                               : cspn3d_gates_bwd_workspace_bytes(B, C, D, H, W, (int)K, (int)prop_step),
                       x);
    if (nd == 2)
        check_rc(cspn2d_gates_bwd_f32(fptr(g), fptr(x), fptr(go), mptr(gg), mptr(gx), B, C, H, W, (int)K, (int)prop_step, ws.ptr(),
                                      ws.bytes, current_stream()),
                 "cspn2d_gates_bwd_f32");
    else
        check_rc(cspn3d_gates_bwd_f32(fptr(g), fptr(x), fptr(go), mptr(gg), mptr(gx), B, C, D, H, W, (int)K, (int)prop_step,
                                      ws.ptr(), ws.bytes, current_stream()),
                 "cspn3d_gates_bwd_f32");
    return {grad_or_empty(gx, x), grad_or_empty(gg, g)};
}

at::Tensor affinity_propagate2d_cuda(const at::Tensor& input, const at::Tensor& gate, int64_t K, int64_t prop_step) {
    return affinity_propagate_cuda(input, gate, K, prop_step, 2);
}
at::Tensor affinity_propagate3d_cuda(const at::Tensor& input, const at::Tensor& gate, int64_t K, int64_t prop_step) {
    return affinity_propagate_cuda(input, gate, K, prop_step, 3);
}
std::tuple<at::Tensor, at::Tensor> affinity_propagate2d_backward_cuda(const at::Tensor& input, const at::Tensor& gate,
                                                                      const at::Tensor& grad_out, int64_t K, int64_t prop_step,
                                                                      bool need_x, bool need_g) {
    return affinity_propagate_backward_cuda(input, gate, grad_out, K, prop_step, need_x, need_g, 2);
}
std::tuple<at::Tensor, at::Tensor> affinity_propagate3d_backward_cuda(const at::Tensor& input, const at::Tensor& gate,
                                                                      const at::Tensor& grad_out, int64_t K, int64_t prop_step,
                                                                      bool need_x, bool need_g) {
    return affinity_propagate_backward_cuda(input, gate, grad_out, K, prop_step, need_x, need_g, 3);
}

// Unpool + crop + 3x3 convolution of the guidance / depth heads: x (B, Cin, h, w), weight (Cout, Cin, 3, 3), out (B, Cout, H, W)
void check_unpool_conv(const at::Tensor& x, const at::Tensor& weight, int64_t H, int64_t W) {
    TORCH_CHECK_VALUE(x.dim() == 4 && weight.dim() == 4 && weight.size(1) == x.size(1) && weight.size(2) == 3 && weight.size(3) == 3,
                      "x must be (B,Cin,h,w) and weight (Cout,Cin,3,3), got ", x.sizes(), " and ", weight.sizes());
    TORCH_CHECK_VALUE(H >= 1 && W >= 1 && H <= 2 * x.size(2) && W <= 2 * x.size(3), "output ", H, "x", W,
                      " must be at least 1x1 and within the unpooled map ", 2 * x.size(2), "x", 2 * x.size(3));
    TORCH_CHECK(x.scalar_type() == at::kFloat && weight.scalar_type() == at::kFloat, "cspn_b200 is fp32 only");
    TORCH_CHECK(x.device() == weight.device(), "x and weight are on different devices");
}

at::Tensor unpool_conv3x3_cuda(const at::Tensor& x, const at::Tensor& weight, int64_t H, int64_t W) {
    check_unpool_conv(x, weight, H, W);
    const c10::cuda::CUDAGuard guard(x.device());
    const at::Tensor xc = x.contiguous(), wc = weight.contiguous();
    at::Tensor out = at::empty({xc.size(0), wc.size(0), H, W}, xc.options());
    check_rc(cspn_unpool_conv3x3_fwd_f32(fptr(xc), fptr(wc), mptr(out), (int)xc.size(0), (int)xc.size(1), (int)xc.size(2),
                                         (int)xc.size(3), (int)wc.size(0), (int)H, (int)W, current_stream()),
             "cspn_unpool_conv3x3_fwd_f32");
    return out;
}

std::tuple<at::Tensor, at::Tensor> unpool_conv3x3_backward_cuda(const at::Tensor& x, const at::Tensor& weight,
                                                                const at::Tensor& grad_out, int64_t H, int64_t W, bool need_x,
                                                                bool need_w) {
    check_unpool_conv(x, weight, H, W);
    TORCH_CHECK(grad_out.dim() == 4 && grad_out.size(0) == x.size(0) && grad_out.size(1) == weight.size(0) && grad_out.size(2) == H &&
                    grad_out.size(3) == W && grad_out.scalar_type() == at::kFloat && grad_out.device() == x.device(),
                "grad_out must be (B,Cout,H,W) fp32 on the device of x, got ", grad_out.sizes());
    const c10::cuda::CUDAGuard guard(x.device());
    const at::Tensor xc = x.contiguous(), wc = weight.contiguous(), go = grad_out.contiguous();
    at::Tensor gx = new_grad(need_x, xc), gw = new_grad(need_w, wc);
    const int B = (int)xc.size(0), Cin = (int)xc.size(1), h = (int)xc.size(2), w = (int)xc.size(3), Cout = (int)wc.size(0);
    const Workspace ws(need_w ? cspn_unpool_conv3x3_bwd_workspace_bytes(B, Cin, h, w, Cout, (int)H, (int)W) : 0, xc);
    if (need_x || need_w)
        check_rc(cspn_unpool_conv3x3_bwd_f32(fptr(xc), fptr(wc), fptr(go), mptr(gx), mptr(gw), B, Cin, h, w, Cout, (int)H, (int)W,
                                             ws.ptr(), ws.bytes, current_stream()),
                 "cspn_unpool_conv3x3_bwd_f32");
    return {grad_or_empty(gx, xc), grad_or_empty(gw, wc)};
}

// a * b * c < 2^31 for non-negative sizes, without overflowing int64
bool volume_fits_int(int64_t a, int64_t b, int64_t c) {
    constexpr int64_t kLimit = (int64_t)1 << 31;
    return a < kLimit && b < kLimit && c < kLimit && a * b < kLimit && a * b * c < kLimit;
}

// Trilinear resampling (the Paddle module's resize_trilinear): (B, C, d, h, w) <-> (B, C, D, H, W)
void check_resize(const at::Tensor& t, int64_t D, int64_t H, int64_t W, int64_t align_mode, const char* name) {
    TORCH_CHECK_VALUE(t.dim() == 5, name, " must be (B,C,D,H,W), got ", t.sizes());
    TORCH_CHECK_VALUE(D >= 1 && H >= 1 && W >= 1, "sizes must be >= 1, got ", D, "x", H, "x", W);
    TORCH_CHECK_VALUE(align_mode == 0 || align_mode == 1, "align_mode must be 0 or 1, got ", align_mode);
    TORCH_CHECK(t.scalar_type() == at::kFloat, "cspn_b200 is fp32 only");
    // the C ABI takes int sizes and < 2^31 elements per (B*C) slice: refuse the rest before allocating or narrowing to int
    TORCH_CHECK(t.size(0) < ((int64_t)1 << 31) && t.size(1) < ((int64_t)1 << 31) && volume_fits_int(t.size(2), t.size(3), t.size(4)) &&
                    volume_fits_int(D, H, W),
                "resize_trilinear takes B, C < 2^31 and < 2^31 elements per (B*C) slice, got ", name, " ", t.sizes(), " and ",
                D, "x", H, "x", W);
}

at::Tensor resize_trilinear_cuda(const at::Tensor& x, int64_t D, int64_t H, int64_t W, bool align_corners, int64_t align_mode) {
    check_resize(x, D, H, W, align_mode, "input");
    const c10::cuda::CUDAGuard guard(x.device());
    const at::Tensor xc = x.contiguous();
    at::Tensor out = at::empty({xc.size(0), xc.size(1), D, H, W}, xc.options());
    if (out.numel())
        check_rc(cspn_resize_trilinear_fwd_f32(fptr(xc), mptr(out), (int)xc.size(0), (int)xc.size(1), (int)xc.size(2),
                                               (int)xc.size(3), (int)xc.size(4), (int)D, (int)H, (int)W, align_corners,
                                               (int)align_mode, current_stream()),
                 "cspn_resize_trilinear_fwd_f32");
    return out;
}

at::Tensor resize_trilinear_backward_cuda(const at::Tensor& grad_out, int64_t D, int64_t H, int64_t W, bool align_corners,
                                          int64_t align_mode) {
    check_resize(grad_out, D, H, W, align_mode, "grad_out");
    const c10::cuda::CUDAGuard guard(grad_out.device());
    const at::Tensor go = grad_out.contiguous();
    at::Tensor gx = at::empty({go.size(0), go.size(1), D, H, W}, go.options());
    const int Do = (int)go.size(2), Ho = (int)go.size(3), Wo = (int)go.size(4);
    if (gx.numel()) {
        const Workspace ws(cspn_resize_trilinear_bwd_workspace_bytes((int)D, (int)H, (int)W, Do, Ho, Wo), go);
        check_rc(cspn_resize_trilinear_bwd_f32(fptr(go), mptr(gx), (int)go.size(0), (int)go.size(1), (int)D, (int)H, (int)W, Do,
                                               Ho, Wo, align_corners, (int)align_mode, ws.ptr(), ws.bytes, current_stream()),
                 "cspn_resize_trilinear_bwd_f32");
    }
    return gx;
}

// Disparity regression (resize_trilinear, softmax over D, expectation): cost (B, C, d, h, w) -> (B, C, H, W)
at::Tensor disparity_regression_cuda(const at::Tensor& cost, int64_t D, int64_t H, int64_t W, bool align_corners,
                                     int64_t align_mode) {
    check_resize(cost, D, H, W, align_mode, "cost");
    const c10::cuda::CUDAGuard guard(cost.device());
    const at::Tensor cc = cost.contiguous();
    at::Tensor out = at::empty({cc.size(0), cc.size(1), H, W}, cc.options());
    if (out.numel())
        check_rc(cspn_disparity_regression_fwd_f32(fptr(cc), mptr(out), (int)cc.size(0), (int)cc.size(1), (int)cc.size(2),
                                                   (int)cc.size(3), (int)cc.size(4), (int)D, (int)H, (int)W, align_corners,
                                                   (int)align_mode, current_stream()),
                 "cspn_disparity_regression_fwd_f32");
    return out;
}

at::Tensor disparity_regression_backward_cuda(const at::Tensor& cost, const at::Tensor& grad_out, int64_t D, int64_t H,
                                              int64_t W, bool align_corners, int64_t align_mode) {
    check_resize(cost, D, H, W, align_mode, "cost");
    TORCH_CHECK_VALUE(grad_out.dim() == 4 && grad_out.size(0) == cost.size(0) && grad_out.size(1) == cost.size(1) &&
                          grad_out.size(2) == H && grad_out.size(3) == W,
                      "grad_out must be (B, C, H, W) = (", cost.size(0), ", ", cost.size(1), ", ", H, ", ", W, "), got ",
                      grad_out.sizes());
    TORCH_CHECK(grad_out.scalar_type() == at::kFloat && grad_out.device() == cost.device(),
                "grad_out must be fp32 on cost's device");
    const c10::cuda::CUDAGuard guard(cost.device());
    const at::Tensor cc = cost.contiguous(), go = grad_out.contiguous();
    at::Tensor gc = at::empty_like(cc);
    if (gc.numel()) {
        const int d = (int)cc.size(2), h = (int)cc.size(3), w = (int)cc.size(4);
        const Workspace ws(cspn_disparity_regression_bwd_workspace_bytes(d, h, w, (int)D, (int)H, (int)W), cc);
        check_rc(cspn_disparity_regression_bwd_f32(fptr(cc), fptr(go), mptr(gc), (int)cc.size(0), (int)cc.size(1), d, h, w,
                                                   (int)D, (int)H, (int)W, align_corners, (int)align_mode, ws.ptr(), ws.bytes,
                                                   current_stream()),
                 "cspn_disparity_regression_bwd_f32");
    }
    return gc;
}

// Stereo cost volumes: left, right (B, F, H, W) -> (B, 2F, D, H, W) (concatenation) or (B, G, D, H, W) (group-wise
// correlation).  The C ABI takes int sizes and < 2^31 elements per (B, channel) slice: refuse the rest before allocating
void check_cost_volume(const at::Tensor& left, const at::Tensor& right, int64_t D, int64_t G) {
    TORCH_CHECK_VALUE(left.dim() == 4 && left.sizes() == right.sizes(), "left and right must be (B,F,H,W) of one shape, got ",
                      left.sizes(), " and ", right.sizes());
    TORCH_CHECK_VALUE(D >= 1, "max_disp must be >= 1, got ", D);
    TORCH_CHECK_VALUE(G >= 1 && left.size(1) % G == 0, "num_groups must be >= 1 and divide F=", left.size(1), ", got ", G);
    TORCH_CHECK(left.scalar_type() == at::kFloat && right.scalar_type() == at::kFloat, "cspn_b200 is fp32 only");
    TORCH_CHECK(left.device() == right.device(), "left and right are on different devices");
    TORCH_CHECK(left.size(0) < ((int64_t)1 << 31) && 2 * left.size(1) < ((int64_t)1 << 31) &&
                    volume_fits_int(D, left.size(2), left.size(3)),
                "the cost volumes take B, 2F < 2^31 and < 2^31 elements per (B, channel) slice, got features ", left.sizes(),
                " and max_disp ", D);
}

at::Tensor concat_volume_cuda(const at::Tensor& left, const at::Tensor& right, int64_t D) {
    check_cost_volume(left, right, D, 1);
    const c10::cuda::CUDAGuard guard(left.device());
    const at::Tensor l = left.contiguous(), r = right.contiguous();
    at::Tensor out = at::empty({l.size(0), 2 * l.size(1), D, l.size(2), l.size(3)}, l.options());
    if (out.numel())
        check_rc(cspn_concat_volume_fwd_f32(fptr(l), fptr(r), mptr(out), (int)l.size(0), (int)l.size(1), (int)l.size(2),
                                            (int)l.size(3), (int)D, current_stream()),
                 "cspn_concat_volume_fwd_f32");
    return out;
}

std::tuple<at::Tensor, at::Tensor> concat_volume_backward_cuda(const at::Tensor& grad_out) {
    TORCH_CHECK_VALUE(grad_out.dim() == 5 && grad_out.size(1) % 2 == 0, "grad_out must be (B,2F,D,H,W), got ", grad_out.sizes());
    TORCH_CHECK(grad_out.scalar_type() == at::kFloat, "cspn_b200 is fp32 only");
    TORCH_CHECK(grad_out.size(0) < ((int64_t)1 << 31) && grad_out.size(1) < ((int64_t)1 << 31) &&
                    volume_fits_int(grad_out.size(2), grad_out.size(3), grad_out.size(4)),
                "the cost volumes take B, 2F < 2^31 and < 2^31 elements per (B, channel) slice, got grad_out ", grad_out.sizes());
    const c10::cuda::CUDAGuard guard(grad_out.device());
    const at::Tensor go = grad_out.contiguous();
    const int64_t B = go.size(0), F = go.size(1) / 2, H = go.size(3), W = go.size(4);
    at::Tensor gl = at::empty({B, F, H, W}, go.options()), gr = at::empty({B, F, H, W}, go.options());
    if (gl.numel() && go.size(2))
        check_rc(cspn_concat_volume_bwd_f32(fptr(go), mptr(gl), mptr(gr), (int)B, (int)F, (int)H, (int)W, (int)go.size(2),
                                            current_stream()),
                 "cspn_concat_volume_bwd_f32");
    return {gl, gr};
}

at::Tensor gwc_volume_cuda(const at::Tensor& left, const at::Tensor& right, int64_t D, int64_t G) {
    check_cost_volume(left, right, D, G);
    const c10::cuda::CUDAGuard guard(left.device());
    const at::Tensor l = left.contiguous(), r = right.contiguous();
    at::Tensor out = at::empty({l.size(0), G, D, l.size(2), l.size(3)}, l.options());
    if (out.numel())
        check_rc(cspn_gwc_volume_fwd_f32(fptr(l), fptr(r), mptr(out), (int)l.size(0), (int)l.size(1), (int)l.size(2),
                                         (int)l.size(3), (int)D, (int)G, current_stream()),
                 "cspn_gwc_volume_fwd_f32");
    return out;
}

std::tuple<at::Tensor, at::Tensor> gwc_volume_backward_cuda(const at::Tensor& left, const at::Tensor& right,
                                                            const at::Tensor& grad_out) {
    TORCH_CHECK_VALUE(grad_out.dim() == 5 && left.dim() == 4 && grad_out.size(0) == left.size(0) &&
                          grad_out.size(3) == left.size(2) && grad_out.size(4) == left.size(3),
                      "grad_out must be (B,G,D,H,W) of left ", left.sizes(), ", got ", grad_out.sizes());
    check_cost_volume(left, right, grad_out.size(2), grad_out.size(1));
    TORCH_CHECK(grad_out.scalar_type() == at::kFloat && grad_out.device() == left.device(), "grad_out must be fp32 on left's device");
    const c10::cuda::CUDAGuard guard(left.device());
    const at::Tensor l = left.contiguous(), r = right.contiguous(), go = grad_out.contiguous();
    at::Tensor gl = at::empty_like(l), gr = at::empty_like(l);
    if (gl.numel())
        check_rc(cspn_gwc_volume_bwd_f32(fptr(l), fptr(r), fptr(go), mptr(gl), mptr(gr), (int)l.size(0), (int)l.size(1),
                                         (int)l.size(2), (int)l.size(3), (int)go.size(2), (int)go.size(1), current_stream()),
                 "cspn_gwc_volume_bwd_f32");
    return {gl, gr};
}

// Affinity pooling: feat (B, C, H, W), gate (B, L, H, W), L kernel sizes -> one flat tensor, level l's (B, C, H/p, W/p)
// after the levels before it.  The C ABI takes int sizes and < 2^31 elements per (B, channel) slice: refuse the rest before
// allocating.  Returns the packed length per (B, channel).
int64_t check_affinity_pool(const at::Tensor& feat, const at::Tensor& gate, at::IntArrayRef ks) {
    TORCH_CHECK_VALUE(feat.dim() == 4 && gate.dim() == 4 && gate.size(0) == feat.size(0) && gate.size(2) == feat.size(2) &&
                          gate.size(3) == feat.size(3),
                      "feat must be (B,C,H,W) and gate (B,L,H,W), got ", feat.sizes(), " and ", gate.sizes());
    TORCH_CHECK_VALUE(ks.size() >= 1 && ks.size() <= 8 && gate.size(1) == (int64_t)ks.size(),
                      "kernel_sizes must hold 1..8 sizes, one per gate channel, got ", ks, " for gate ", gate.sizes());
    TORCH_CHECK(feat.scalar_type() == at::kFloat && gate.scalar_type() == at::kFloat, "cspn_b200 is fp32 only");
    TORCH_CHECK(feat.device() == gate.device(), "feat and gate are on different devices");
    const int64_t H = feat.size(2), W = feat.size(3);
    TORCH_CHECK_VALUE(feat.numel() > 0, "feat must not be empty, got ", feat.sizes());
    int64_t n = 0;
    for (int64_t p : ks) {
        TORCH_CHECK_VALUE(p >= 1 && p <= std::min(H, W), "kernel sizes must be in [1, min(H, W)], got ", ks, " for ", H, "x", W);
        n += (H / p) * (W / p);
    }
    TORCH_CHECK(feat.size(0) < ((int64_t)1 << 31) && feat.size(1) < ((int64_t)1 << 31) && volume_fits_int(1, H, W),
                "affinity_pool2d takes B, C < 2^31 and < 2^31 elements per (B, channel) slice, got feat ", feat.sizes());
    return n;
}

std::vector<int> int_sizes(at::IntArrayRef ks) { return std::vector<int>(ks.begin(), ks.end()); }

at::Tensor affinity_pool2d_cuda(const at::Tensor& feat, const at::Tensor& gate, at::IntArrayRef ks) {
    const int64_t n = check_affinity_pool(feat, gate, ks);
    const c10::cuda::CUDAGuard guard(feat.device());
    const at::Tensor f = feat.contiguous(), g = gate.contiguous();
    at::Tensor out = at::empty({f.size(0) * f.size(1) * n}, f.options());
    const std::vector<int> k = int_sizes(ks);
    check_rc(cspn_affinity_pool2d_fwd_f32(fptr(f), fptr(g), mptr(out), (int)f.size(0), (int)f.size(1), (int)f.size(2),
                                          (int)f.size(3), (int)k.size(), k.data(), current_stream()),
             "cspn_affinity_pool2d_fwd_f32");
    return out;
}

std::tuple<at::Tensor, at::Tensor> affinity_pool2d_backward_cuda(const at::Tensor& feat, const at::Tensor& gate,
                                                                 const at::Tensor& out, const at::Tensor& grad_out,
                                                                 at::IntArrayRef ks) {
    const int64_t n = check_affinity_pool(feat, gate, ks);
    const int64_t len = feat.size(0) * feat.size(1) * n;
    TORCH_CHECK_VALUE(out.dim() == 1 && out.size(0) == len && grad_out.dim() == 1 && grad_out.size(0) == len,
                      "out and grad_out must be the packed levels (", len, "), got ", out.sizes(), " and ", grad_out.sizes());
    TORCH_CHECK(out.scalar_type() == at::kFloat && grad_out.scalar_type() == at::kFloat && out.device() == feat.device() &&
                    grad_out.device() == feat.device(),
                "out and grad_out must be fp32 on feat's device");
    const c10::cuda::CUDAGuard guard(feat.device());
    const at::Tensor f = feat.contiguous(), g = gate.contiguous(), o = out.contiguous(), go = grad_out.contiguous();
    at::Tensor gf = at::empty_like(f), gg = at::empty_like(g);
    const std::vector<int> k = int_sizes(ks);
    check_rc(cspn_affinity_pool2d_bwd_f32(fptr(f), fptr(g), fptr(o), fptr(go), mptr(gf), mptr(gg), (int)f.size(0), (int)f.size(1),
                                          (int)f.size(2), (int)f.size(3), (int)k.size(), k.data(), current_stream()),
             "cspn_affinity_pool2d_bwd_f32");
    return {gf, gg};
}

// Affinity fusion: L levels (B, C, h_l, w_l) and gate (B, L, H, W) -> (B, C, H, W).  The C ABI takes int sizes and < 2^31
// elements per (B, channel) slice of every tensor: refuse the rest before allocating or narrowing to int.  Returns the
// levels' (h_l, w_l), flattened.
std::vector<int> check_affinity_fuse(at::TensorList levels, const at::Tensor& gate, int64_t align_mode) {
    TORCH_CHECK_VALUE(levels.size() >= 1 && levels.size() <= 8, "levels must hold 1..8 tensors, got ", levels.size());
    TORCH_CHECK_VALUE(gate.dim() == 4 && gate.size(1) == (int64_t)levels.size(),
                      "gate must be (B, L, H, W) with L = ", levels.size(), " levels, got ", gate.sizes());
    TORCH_CHECK_VALUE(align_mode == 0 || align_mode == 1, "align_mode must be 0 or 1, got ", align_mode);
    TORCH_CHECK_VALUE(gate.numel() > 0, "gate must not be empty, got ", gate.sizes());
    const at::Tensor& x0 = levels[0];
    TORCH_CHECK(gate.scalar_type() == at::kFloat, "cspn_b200 is fp32 only");
    std::vector<int> hw;
    for (const at::Tensor& x : levels) {
        TORCH_CHECK_VALUE(x.dim() == 4 && x.size(0) == gate.size(0) && x.size(1) == x0.size(1) && x.numel() > 0,
                          "every level must be a non-empty (B, C, h, w) with gate's B and one C, got ", x.sizes(), " for gate ",
                          gate.sizes());
        TORCH_CHECK(x.scalar_type() == at::kFloat, "cspn_b200 is fp32 only");
        TORCH_CHECK(x.device() == gate.device(), "the levels and gate are on different devices");
        TORCH_CHECK(volume_fits_int(1, x.size(2), x.size(3)), "affinity_fuse2d takes < 2^31 elements per (B, channel) slice, got ",
                    x.sizes());
        hw.push_back((int)x.size(2));
        hw.push_back((int)x.size(3));
    }
    TORCH_CHECK(gate.size(0) < ((int64_t)1 << 31) && x0.size(1) < ((int64_t)1 << 31) && volume_fits_int(1, gate.size(2), gate.size(3)),
                "affinity_fuse2d takes B, C < 2^31 and < 2^31 elements per (B, channel) slice, got gate ", gate.sizes());
    return hw;
}

std::vector<const float*> level_ptrs(const std::vector<at::Tensor>& xs) {
    std::vector<const float*> p;
    for (const at::Tensor& x : xs) p.push_back(fptr(x));
    return p;
}

std::vector<at::Tensor> contiguous_all(at::TensorList xs) {
    std::vector<at::Tensor> c;
    for (const at::Tensor& x : xs) c.push_back(x.contiguous());
    return c;
}

at::Tensor affinity_fuse2d_cuda(at::TensorList levels, const at::Tensor& gate, bool align_corners, int64_t align_mode) {
    const std::vector<int> hw = check_affinity_fuse(levels, gate, align_mode);
    const c10::cuda::CUDAGuard guard(gate.device());
    const std::vector<at::Tensor> xs = contiguous_all(levels);
    const at::Tensor g = gate.contiguous();
    at::Tensor out = at::empty({g.size(0), xs[0].size(1), g.size(2), g.size(3)}, g.options());
    check_rc(cspn_affinity_fuse2d_fwd_f32(level_ptrs(xs).data(), hw.data(), fptr(g), mptr(out), (int)g.size(0), (int)xs[0].size(1),
                                          (int)g.size(2), (int)g.size(3), (int)xs.size(), align_corners, (int)align_mode,
                                          current_stream()),
             "cspn_affinity_fuse2d_fwd_f32");
    return out;
}

std::tuple<std::vector<at::Tensor>, at::Tensor> affinity_fuse2d_backward_cuda(at::TensorList levels, const at::Tensor& gate,
                                                                              const at::Tensor& out, const at::Tensor& grad_out,
                                                                              bool align_corners, int64_t align_mode) {
    const std::vector<int> hw = check_affinity_fuse(levels, gate, align_mode);
    const std::vector<int64_t> shape{gate.size(0), levels[0].size(1), gate.size(2), gate.size(3)};
    TORCH_CHECK_VALUE(out.sizes() == at::IntArrayRef(shape) && grad_out.sizes() == at::IntArrayRef(shape),
                      "out and grad_out must be (B, C, H, W) = ", at::IntArrayRef(shape), ", got ", out.sizes(), " and ",
                      grad_out.sizes());
    TORCH_CHECK(out.scalar_type() == at::kFloat && grad_out.scalar_type() == at::kFloat && out.device() == gate.device() &&
                    grad_out.device() == gate.device(),
                "out and grad_out must be fp32 on gate's device");
    const c10::cuda::CUDAGuard guard(gate.device());
    const std::vector<at::Tensor> xs = contiguous_all(levels);
    const at::Tensor g = gate.contiguous(), o = out.contiguous(), go = grad_out.contiguous();
    std::vector<at::Tensor> gl;
    std::vector<float*> glp;
    for (const at::Tensor& x : xs) {
        gl.push_back(at::empty_like(x));
        glp.push_back(mptr(gl.back()));
    }
    at::Tensor gg = at::empty_like(g);
    const int B = (int)g.size(0), C = (int)xs[0].size(1), H = (int)g.size(2), W = (int)g.size(3), L = (int)xs.size();
    const Workspace ws(cspn_affinity_fuse2d_bwd_workspace_bytes(B, C, H, W, L, hw.data()), g);
    check_rc(cspn_affinity_fuse2d_bwd_f32(level_ptrs(xs).data(), hw.data(), fptr(g), fptr(o), fptr(go), glp.data(), mptr(gg), B, C,
                                          H, W, L, align_corners, (int)align_mode, ws.ptr(), ws.bytes, current_stream()),
             "cspn_affinity_fuse2d_bwd_f32");
    return {gl, gg};
}

// Atrous affinity pooling: feat (B, C, H, W), gate (B, 9L, H, W), L rates -> (B, L*C, H, W).  The C ABI takes int sizes and
// < 2^31 elements per (B, channel) slice: refuse the rest before allocating or narrowing to int.
void check_affinity_atrous(const at::Tensor& feat, const at::Tensor& gate, at::IntArrayRef rates) {
    TORCH_CHECK_VALUE(feat.dim() == 4 && gate.dim() == 4 && gate.size(0) == feat.size(0) && gate.size(2) == feat.size(2) &&
                          gate.size(3) == feat.size(3),
                      "feat must be (B,C,H,W) and gate (B,9L,H,W), got ", feat.sizes(), " and ", gate.sizes());
    TORCH_CHECK_VALUE(rates.size() >= 1 && rates.size() <= 8 && gate.size(1) == 9 * (int64_t)rates.size(),
                      "dilations must hold 1..8 rates, nine gate channels each, got ", rates, " for gate ", gate.sizes());
    TORCH_CHECK(feat.scalar_type() == at::kFloat && gate.scalar_type() == at::kFloat, "cspn_b200 is fp32 only");
    TORCH_CHECK(feat.device() == gate.device(), "feat and gate are on different devices");
    const int64_t H = feat.size(2), W = feat.size(3);
    TORCH_CHECK_VALUE(feat.numel() > 0, "feat must not be empty, got ", feat.sizes());
    for (int64_t r : rates)
        TORCH_CHECK_VALUE(r >= 1 && r <= std::max(H, W), "dilations must be in [1, max(H, W)], got ", rates, " for ", H, "x", W);
    TORCH_CHECK(feat.size(0) < ((int64_t)1 << 31) && feat.size(1) < ((int64_t)1 << 31) && volume_fits_int(1, H, W),
                "affinity_atrous_pool2d takes B, C < 2^31 and < 2^31 elements per (B, channel) slice, got feat ", feat.sizes());
}

at::Tensor affinity_atrous_pool2d_cuda(const at::Tensor& feat, const at::Tensor& gate, at::IntArrayRef rates) {
    check_affinity_atrous(feat, gate, rates);
    const c10::cuda::CUDAGuard guard(feat.device());
    const at::Tensor f = feat.contiguous(), g = gate.contiguous();
    at::Tensor out = at::empty({f.size(0), (int64_t)rates.size() * f.size(1), f.size(2), f.size(3)}, f.options());
    const std::vector<int> r = int_sizes(rates);
    check_rc(cspn_affinity_atrous2d_fwd_f32(fptr(f), fptr(g), mptr(out), (int)f.size(0), (int)f.size(1), (int)f.size(2),
                                            (int)f.size(3), (int)r.size(), r.data(), current_stream()),
             "cspn_affinity_atrous2d_fwd_f32");
    return out;
}

std::tuple<at::Tensor, at::Tensor> affinity_atrous_pool2d_backward_cuda(const at::Tensor& feat, const at::Tensor& gate,
                                                                        const at::Tensor& out, const at::Tensor& grad_out,
                                                                        at::IntArrayRef rates) {
    check_affinity_atrous(feat, gate, rates);
    const std::vector<int64_t> shape{feat.size(0), (int64_t)rates.size() * feat.size(1), feat.size(2), feat.size(3)};
    TORCH_CHECK_VALUE(out.sizes() == at::IntArrayRef(shape) && grad_out.sizes() == at::IntArrayRef(shape),
                      "out and grad_out must be (B, L*C, H, W) = ", at::IntArrayRef(shape), ", got ", out.sizes(), " and ",
                      grad_out.sizes());
    TORCH_CHECK(out.scalar_type() == at::kFloat && grad_out.scalar_type() == at::kFloat && out.device() == feat.device() &&
                    grad_out.device() == feat.device(),
                "out and grad_out must be fp32 on feat's device");
    const c10::cuda::CUDAGuard guard(feat.device());
    const at::Tensor f = feat.contiguous(), g = gate.contiguous(), o = out.contiguous(), go = grad_out.contiguous();
    at::Tensor gf = at::empty_like(f), gg = at::empty_like(g);
    const std::vector<int> r = int_sizes(rates);
    const int B = (int)f.size(0), C = (int)f.size(1), H = (int)f.size(2), W = (int)f.size(3), L = (int)r.size();
    const Workspace ws(cspn_affinity_atrous2d_bwd_workspace_bytes(B, C, H, W, L, r.data()), f);
    check_rc(cspn_affinity_atrous2d_bwd_f32(fptr(f), fptr(g), fptr(o), fptr(go), mptr(gf), mptr(gg), B, C, H, W, L, r.data(),
                                            ws.ptr(), ws.bytes, current_stream()),
             "cspn_affinity_atrous2d_bwd_f32");
    return {gf, gg};
}

}  // namespace

TORCH_LIBRARY(cspn_b200, m) {
    m.def("propagate2d(Tensor guidance, Tensor blur_depth, Tensor? sparse_depth, int prop_time, int norm_type, int algo) -> Tensor");
    m.def("propagate2d_backward(Tensor guidance, Tensor blur_depth, Tensor? sparse_depth, Tensor grad_out, int prop_time, "
          "int norm_type, bool need_guidance, bool need_blur) -> (Tensor, Tensor)");
    m.def("propagate2d_k(Tensor guidance, Tensor blur_depth, Tensor? sparse_depth, int kernel_size, int prop_time, "
          "int norm_type) -> Tensor");
    m.def("propagate2d_k_backward(Tensor guidance, Tensor blur_depth, Tensor? sparse_depth, Tensor grad_out, int kernel_size, "
          "int prop_time, int norm_type, bool need_guidance, bool need_blur) -> (Tensor, Tensor)");
    m.def("propagate2d_keep(Tensor guidance, Tensor blur_depth, Tensor? sparse_depth, int kernel_size, int prop_time, "
          "int norm_type, int algo) -> Tensor");
    m.def("propagate2d_keep_backward(Tensor guidance, Tensor blur_depth, Tensor? sparse_depth, Tensor grad_out, int kernel_size, "
          "int prop_time, int norm_type, bool need_guidance, bool need_blur, bool need_sparse) -> (Tensor, Tensor, Tensor)");
    m.def("propagate2d_aggregate(Tensor guidance, Tensor blur_depth, Tensor? sparse_depth, Tensor step_weight, int[] steps, "
          "int kernel_size, int norm_type, bool keep) -> Tensor");
    m.def("propagate2d_aggregate_backward(Tensor guidance, Tensor blur_depth, Tensor? sparse_depth, Tensor step_weight, "
          "Tensor grad_out, int[] steps, int kernel_size, int norm_type, bool keep, bool need_guidance, bool need_blur, "
          "bool need_sparse, bool need_step_weight) -> (Tensor, Tensor, Tensor, Tensor)");
    m.def("propagate2d_nonlocal(Tensor feat, Tensor offset, Tensor affinity, Tensor? sparse_depth, int kernel_size, int prop_time) "
          "-> Tensor");
    m.def("propagate2d_nonlocal_backward(Tensor feat, Tensor offset, Tensor affinity, Tensor? sparse_depth, Tensor grad_out, "
          "int kernel_size, int prop_time, bool need_feat, bool need_offset, bool need_affinity, bool need_sparse) -> "
          "(Tensor, Tensor, Tensor, Tensor)");
    m.def("propagate2d_dilated(Tensor kernel, Tensor blur_depth, Tensor? sparse_depth, Tensor? confidence, int kernel_size, "
          "int dilation, int prop_time) -> Tensor");
    m.def("propagate2d_dilated_backward(Tensor kernel, Tensor blur_depth, Tensor? sparse_depth, Tensor? confidence, Tensor grad_out, "
          "int kernel_size, int dilation, int prop_time, bool need_kernel, bool need_blur, bool need_sparse, bool need_confidence) -> "
          "(Tensor, Tensor, Tensor, Tensor)");
    m.def("propagate2d_dynamic(Tensor affinity, Tensor attention, Tensor blur_depth, Tensor? sparse_depth, Tensor? confidence, "
          "int kernel_size) -> Tensor");
    m.def("propagate2d_dynamic_backward(Tensor affinity, Tensor attention, Tensor blur_depth, Tensor? sparse_depth, Tensor? confidence, "
          "Tensor grad_out, int kernel_size, bool need_affinity, bool need_attention, bool need_blur, bool need_sparse, "
          "bool need_confidence) -> (Tensor, Tensor, Tensor, Tensor, Tensor)");
    m.def("propagate2d_linear(Tensor feat, Tensor gate, int dir_mask) -> (Tensor, Tensor)");
    m.def("propagate2d_linear_backward(Tensor feat, Tensor gate, Tensor planes, Tensor grad_out, int dir_mask, bool need_feat, "
          "bool need_gate) -> (Tensor, Tensor)");
    m.def("propagate2d_paddle(Tensor guidance, Tensor feat, int kernel_size, int prop_time) -> Tensor");
    m.def("propagate2d_paddle_backward(Tensor guidance, Tensor feat, Tensor grad_out, int kernel_size, int prop_time, "
          "bool need_guidance, bool need_feat) -> (Tensor, Tensor)");
    m.def("propagate3d(Tensor guidance, Tensor feat, int prop_time, int norm_type) -> Tensor");
    m.def("propagate3d_backward(Tensor guidance, Tensor feat, Tensor grad_out, int prop_time, int norm_type, "
          "bool need_guidance, bool need_feat) -> (Tensor, Tensor)");
    m.def("propagate3d_k(Tensor guidance, Tensor feat, int kernel_size, int prop_time, int norm_type) -> Tensor");
    m.def("propagate3d_k_backward(Tensor guidance, Tensor feat, Tensor grad_out, int kernel_size, int prop_time, int norm_type, "
          "bool need_guidance, bool need_feat) -> (Tensor, Tensor)");
    m.def("affinity_propagate2d(Tensor input, Tensor gate_weight, int kernel_size, int prop_step) -> Tensor");
    m.def("affinity_propagate2d_backward(Tensor input, Tensor gate_weight, Tensor grad_out, int kernel_size, int prop_step, "
          "bool need_input, bool need_gate) -> (Tensor, Tensor)");
    m.def("affinity_propagate3d(Tensor input, Tensor gate_weight, int kernel_size, int prop_step) -> Tensor");
    m.def("affinity_propagate3d_backward(Tensor input, Tensor gate_weight, Tensor grad_out, int kernel_size, int prop_step, "
          "bool need_input, bool need_gate) -> (Tensor, Tensor)");
    m.def("unpool_conv3x3(Tensor x, Tensor weight, int H, int W) -> Tensor");
    m.def("unpool_conv3x3_backward(Tensor x, Tensor weight, Tensor grad_out, int H, int W, bool need_x, bool need_weight) "
          "-> (Tensor, Tensor)");
    m.def("resize_trilinear(Tensor input, int D, int H, int W, bool align_corners, int align_mode) -> Tensor");
    m.def("resize_trilinear_backward(Tensor grad_out, int in_D, int in_H, int in_W, bool align_corners, int align_mode) -> Tensor");
    m.def("disparity_regression(Tensor cost, int D, int H, int W, bool align_corners, int align_mode) -> Tensor");
    m.def("disparity_regression_backward(Tensor cost, Tensor grad_out, int D, int H, int W, bool align_corners, int align_mode) "
          "-> Tensor");
    m.def("concat_volume(Tensor left, Tensor right, int max_disp) -> Tensor");
    m.def("concat_volume_backward(Tensor grad_out) -> (Tensor, Tensor)");
    m.def("gwc_volume(Tensor left, Tensor right, int max_disp, int num_groups) -> Tensor");
    m.def("gwc_volume_backward(Tensor left, Tensor right, Tensor grad_out) -> (Tensor, Tensor)");
    m.def("affinity_pool2d(Tensor feat, Tensor gate, int[] kernel_sizes) -> Tensor");
    m.def("affinity_pool2d_backward(Tensor feat, Tensor gate, Tensor out, Tensor grad_out, int[] kernel_sizes) -> (Tensor, Tensor)");
    m.def("affinity_fuse2d(Tensor[] levels, Tensor gate, bool align_corners, int align_mode) -> Tensor");
    m.def("affinity_fuse2d_backward(Tensor[] levels, Tensor gate, Tensor out, Tensor grad_out, bool align_corners, "
          "int align_mode) -> (Tensor[], Tensor)");
    m.def("affinity_atrous_pool2d(Tensor feat, Tensor gate, int[] dilations) -> Tensor");
    m.def("affinity_atrous_pool2d_backward(Tensor feat, Tensor gate, Tensor out, Tensor grad_out, int[] dilations) -> "
          "(Tensor, Tensor)");
}

TORCH_LIBRARY_IMPL(cspn_b200, CUDA, m) {
    m.impl("propagate2d", &propagate2d_cuda);
    m.impl("propagate2d_backward", &propagate2d_backward_cuda);
    m.impl("propagate2d_k", &propagate2d_k_cuda);
    m.impl("propagate2d_k_backward", &propagate2d_k_backward_cuda);
    m.impl("propagate2d_keep", &propagate2d_keep_cuda);
    m.impl("propagate2d_keep_backward", &propagate2d_keep_backward_cuda);
    m.impl("propagate2d_aggregate", &propagate2d_aggregate_cuda);
    m.impl("propagate2d_aggregate_backward", &propagate2d_aggregate_backward_cuda);
    m.impl("propagate2d_nonlocal", &propagate2d_nonlocal_cuda);
    m.impl("propagate2d_nonlocal_backward", &propagate2d_nonlocal_backward_cuda);
    m.impl("propagate2d_dilated", &propagate2d_dilated_cuda);
    m.impl("propagate2d_dilated_backward", &propagate2d_dilated_backward_cuda);
    m.impl("propagate2d_dynamic", &propagate2d_dynamic_cuda);
    m.impl("propagate2d_dynamic_backward", &propagate2d_dynamic_backward_cuda);
    m.impl("propagate2d_linear", &propagate2d_linear_cuda);
    m.impl("propagate2d_linear_backward", &propagate2d_linear_backward_cuda);
    m.impl("propagate2d_paddle", &propagate2d_paddle_cuda);
    m.impl("propagate2d_paddle_backward", &propagate2d_paddle_backward_cuda);
    m.impl("propagate3d", &propagate3d_cuda);
    m.impl("propagate3d_backward", &propagate3d_backward_cuda);
    m.impl("propagate3d_k", &propagate3d_k_cuda);
    m.impl("propagate3d_k_backward", &propagate3d_k_backward_cuda);
    m.impl("affinity_propagate2d", &affinity_propagate2d_cuda);
    m.impl("affinity_propagate2d_backward", &affinity_propagate2d_backward_cuda);
    m.impl("affinity_propagate3d", &affinity_propagate3d_cuda);
    m.impl("affinity_propagate3d_backward", &affinity_propagate3d_backward_cuda);
    m.impl("unpool_conv3x3", &unpool_conv3x3_cuda);
    m.impl("unpool_conv3x3_backward", &unpool_conv3x3_backward_cuda);
    m.impl("resize_trilinear", &resize_trilinear_cuda);
    m.impl("resize_trilinear_backward", &resize_trilinear_backward_cuda);
    m.impl("disparity_regression", &disparity_regression_cuda);
    m.impl("disparity_regression_backward", &disparity_regression_backward_cuda);
    m.impl("concat_volume", &concat_volume_cuda);
    m.impl("concat_volume_backward", &concat_volume_backward_cuda);
    m.impl("gwc_volume", &gwc_volume_cuda);
    m.impl("gwc_volume_backward", &gwc_volume_backward_cuda);
    m.impl("affinity_pool2d", &affinity_pool2d_cuda);
    m.impl("affinity_pool2d_backward", &affinity_pool2d_backward_cuda);
    m.impl("affinity_fuse2d", &affinity_fuse2d_cuda);
    m.impl("affinity_fuse2d_backward", &affinity_fuse2d_backward_cuda);
    m.impl("affinity_atrous_pool2d", &affinity_atrous_pool2d_cuda);
    m.impl("affinity_atrous_pool2d_backward", &affinity_atrous_pool2d_backward_cuda);
}
