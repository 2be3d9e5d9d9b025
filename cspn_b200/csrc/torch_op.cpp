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
// There is no CPU kernel: CPU tensors reach the dispatcher's "no kernel for backend CPU" error, loudly.
#include <ATen/ATen.h>
#include <c10/cuda/CUDAGuard.h>
#include <c10/cuda/CUDAStream.h>
#include <torch/library.h>

#include <optional>
#include <tuple>
#include <utility>

#include "../../include/cspn_b200.h"

namespace {

const float* fptr(const at::Tensor& t) { return t.data_ptr<float>(); }

void check_rc(int rc, const char* what) {
    if (rc == CSPN_OK) return;
    const char* msg = cspn_last_error();
    TORCH_CHECK(rc != CSPN_ERR_INVALID_ARGUMENT, what, ": ", msg);
    TORCH_CHECK(false, what, " failed (status ", rc, "): ", msg);
}

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
    const size_t ws_bytes = cspn2d_workspace_bytes(B, C, H, W, (int)prop_time, a);
    at::Tensor ws;
    if (ws_bytes) ws = at::empty({(int64_t)ws_bytes}, d.options().dtype(at::kByte));
    check_rc(cspn2d_fwd_f32(fptr(g), fptr(d), s.defined() ? fptr(s) : nullptr, out.data_ptr<float>(), B, C, H, W, (int)g.size(1),
                            (int)prop_time, (int)norm_type, a, ws_bytes ? ws.data_ptr() : nullptr, ws_bytes,
                            (cspn_stream_t)c10::cuda::getCurrentCUDAStream().stream()),
             "cspn2d_fwd_f32");
    return out;
}

std::tuple<at::Tensor, at::Tensor> propagate2d_backward_cuda(const at::Tensor& guidance, const at::Tensor& blur,
                                                             const std::optional<at::Tensor>& sparse, const at::Tensor& grad_out,
                                                             int64_t prop_time, int64_t norm_type, bool need_g, bool need_d) {
    check2d(guidance, blur, sparse);
    TORCH_CHECK(grad_out.sizes() == blur.sizes() && grad_out.scalar_type() == at::kFloat && grad_out.device() == blur.device(),
                "grad_out must match blur_depth");
    const c10::cuda::CUDAGuard guard(blur.device());
    const at::Tensor g = guidance.contiguous(), d = blur.contiguous(), go = grad_out.contiguous();
    const at::Tensor s = sparse.has_value() ? sparse->contiguous() : at::Tensor();
    at::Tensor gg = need_g ? at::empty_like(g) : at::Tensor();
    at::Tensor gd = need_d ? at::empty_like(d) : at::Tensor();
    if (prop_time == 0) {                              // identity: d out / d blur = 1, no dependence on the guidance
        if (need_g) gg.zero_();
        if (need_d) gd.copy_(go);
        return {need_g ? gg : at::zeros({0}, g.options()), need_d ? gd : at::zeros({0}, d.options())};
    }
    const int B = (int)d.size(0), C = (int)d.size(1), H = (int)d.size(2), W = (int)d.size(3);
    const size_t ws_bytes = cspn2d_bwd_workspace_bytes(B, C, H, W, (int)prop_time);
    at::Tensor ws;
    if (ws_bytes) ws = at::empty({(int64_t)ws_bytes}, d.options().dtype(at::kByte));
    check_rc(cspn2d_bwd_f32(fptr(g), fptr(d), s.defined() ? fptr(s) : nullptr, fptr(go), need_g ? gg.data_ptr<float>() : nullptr,
                            need_d ? gd.data_ptr<float>() : nullptr, B, C, H, W, (int)g.size(1), (int)prop_time, (int)norm_type,
                            ws_bytes ? ws.data_ptr() : nullptr, ws_bytes, (cspn_stream_t)c10::cuda::getCurrentCUDAStream().stream()),
             "cspn2d_bwd_f32");
    // an unused gradient is returned as an empty tensor (the Python autograd formula maps it to None)
    return {need_g ? gg : at::zeros({0}, g.options()), need_d ? gd : at::zeros({0}, d.options())};
}

// K x K kernels: K = 3 is the 3x3 operator above (same kernels, same bits); K = 5 / 7 go through cspn2d_k_*_f32
void check2d_k(const at::Tensor& guidance, const at::Tensor& blur, const std::optional<at::Tensor>& sparse, int64_t K) {
    TORCH_CHECK(K == 3 || K == 5 || K == 7, "kernel_size must be 3, 5 or 7, got ", K);
    check2d(guidance, blur, sparse);
    TORCH_CHECK(guidance.size(1) >= K * K - 1, "a ", K, "x", K, " kernel needs guidance (B,>=", K * K - 1, ",H,W), got ",
                guidance.sizes());
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
    const size_t ws_bytes = cspn2d_k_workspace_bytes(B, C, H, W, (int)K, (int)prop_time);
    at::Tensor ws;
    if (ws_bytes) ws = at::empty({(int64_t)ws_bytes}, d.options().dtype(at::kByte));
    check_rc(cspn2d_k_fwd_f32(fptr(g), fptr(d), s.defined() ? fptr(s) : nullptr, out.data_ptr<float>(), B, C, H, W,
                              (int)g.size(1), (int)K, (int)prop_time, (int)norm_type, ws_bytes ? ws.data_ptr() : nullptr,
                              ws_bytes, (cspn_stream_t)c10::cuda::getCurrentCUDAStream().stream()),
             "cspn2d_k_fwd_f32");
    return out;
}

std::tuple<at::Tensor, at::Tensor> propagate2d_k_backward_cuda(const at::Tensor& guidance, const at::Tensor& blur,
                                                               const std::optional<at::Tensor>& sparse, const at::Tensor& grad_out,
                                                               int64_t K, int64_t prop_time, int64_t norm_type, bool need_g,
                                                               bool need_d) {
    check2d_k(guidance, blur, sparse, K);
    if (K == 3) return propagate2d_backward_cuda(guidance, blur, sparse, grad_out, prop_time, norm_type, need_g, need_d);
    TORCH_CHECK(grad_out.sizes() == blur.sizes() && grad_out.scalar_type() == at::kFloat && grad_out.device() == blur.device(),
                "grad_out must match blur_depth");
    const c10::cuda::CUDAGuard guard(blur.device());
    const at::Tensor g = guidance.contiguous(), d = blur.contiguous(), go = grad_out.contiguous();
    const at::Tensor s = sparse.has_value() ? sparse->contiguous() : at::Tensor();
    at::Tensor gg = need_g ? at::empty_like(g) : at::Tensor();
    at::Tensor gd = need_d ? at::empty_like(d) : at::Tensor();
    const int B = (int)d.size(0), C = (int)d.size(1), H = (int)d.size(2), W = (int)d.size(3);
    const size_t ws_bytes = cspn2d_k_bwd_workspace_bytes(B, C, H, W, (int)K, (int)prop_time);
    at::Tensor ws;
    if (ws_bytes) ws = at::empty({(int64_t)ws_bytes}, d.options().dtype(at::kByte));
    check_rc(cspn2d_k_bwd_f32(fptr(g), fptr(d), s.defined() ? fptr(s) : nullptr, fptr(go), need_g ? gg.data_ptr<float>() : nullptr,
                              need_d ? gd.data_ptr<float>() : nullptr, B, C, H, W, (int)g.size(1), (int)K, (int)prop_time,
                              (int)norm_type, ws_bytes ? ws.data_ptr() : nullptr, ws_bytes,
                              (cspn_stream_t)c10::cuda::getCurrentCUDAStream().stream()),
             "cspn2d_k_bwd_f32");
    return {need_g ? gg : at::zeros({0}, g.options()), need_d ? gd : at::zeros({0}, d.options())};
}

// 2D 'paddle' (own-location gates), K in {3, 5, 7}.  guidance (B, K*K-1, H, W) is shared by the C channels of feat;
// (B, (K*K-1)*C, H, W) with C > 1 gives channel c its own gate (demo.py:28-45), which in memory is B*C images of one
// channel.  Returns the (images, channels) the C ABI is called with.
std::pair<int, int> check2d_paddle(const at::Tensor& guidance, const at::Tensor& feat, int64_t K) {
    TORCH_CHECK_VALUE(K == 3 || K == 5 || K == 7, "kernel_size must be 3, 5 or 7, got ", K);
    TORCH_CHECK_VALUE(guidance.dim() == 4 && feat.dim() == 4, "guidance and feat must be (B,C,H,W)");
    TORCH_CHECK(guidance.scalar_type() == at::kFloat && feat.scalar_type() == at::kFloat, "cspn_b200 is fp32 only");
    const int64_t nt = K * K - 1, B = feat.size(0), C = feat.size(1);
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
    const size_t ws_bytes = cspn2d_paddle_workspace_bytes(B, C, H, W, (int)K, (int)prop_time);
    at::Tensor ws;
    if (ws_bytes) ws = at::empty({(int64_t)ws_bytes}, f.options().dtype(at::kByte));
    check_rc(cspn2d_paddle_fwd_f32(fptr(g), fptr(f), out.data_ptr<float>(), B, C, H, W, (int)K, (int)prop_time,
                                   ws_bytes ? ws.data_ptr() : nullptr, ws_bytes, (cspn_stream_t)c10::cuda::getCurrentCUDAStream().stream()),
             "cspn2d_paddle_fwd_f32");
    return out;
}

std::tuple<at::Tensor, at::Tensor> propagate2d_paddle_backward_cuda(const at::Tensor& guidance, const at::Tensor& feat,
                                                                    const at::Tensor& grad_out, int64_t K, int64_t prop_time,
                                                                    bool need_g, bool need_f) {
    const auto [B, C] = check2d_paddle(guidance, feat, K);
    TORCH_CHECK(grad_out.sizes() == feat.sizes() && grad_out.scalar_type() == at::kFloat && grad_out.device() == feat.device(),
                "grad_out must match feat");
    const c10::cuda::CUDAGuard guard(feat.device());
    const at::Tensor g = guidance.contiguous(), f = feat.contiguous(), go = grad_out.contiguous();
    at::Tensor gg = need_g ? at::empty_like(g) : at::Tensor();
    at::Tensor gf = need_f ? at::empty_like(f) : at::Tensor();
    const int H = (int)f.size(2), W = (int)f.size(3);
    const size_t ws_bytes = cspn2d_paddle_bwd_workspace_bytes(B, C, H, W, (int)K, (int)prop_time);
    at::Tensor ws;
    if (ws_bytes) ws = at::empty({(int64_t)ws_bytes}, f.options().dtype(at::kByte));
    check_rc(cspn2d_paddle_bwd_f32(fptr(g), fptr(f), fptr(go), need_g ? gg.data_ptr<float>() : nullptr,
                                   need_f ? gf.data_ptr<float>() : nullptr, B, C, H, W, (int)K, (int)prop_time,
                                   ws_bytes ? ws.data_ptr() : nullptr, ws_bytes, (cspn_stream_t)c10::cuda::getCurrentCUDAStream().stream()),
             "cspn2d_paddle_bwd_f32");
    return {need_g ? gg : at::zeros({0}, g.options()), need_f ? gf : at::zeros({0}, f.options())};
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
    const size_t ws_bytes = cspn3d_workspace_bytes(B, C, D, H, W, (int)prop_time);
    at::Tensor ws;
    if (ws_bytes) ws = at::empty({(int64_t)ws_bytes}, f.options().dtype(at::kByte));
    check_rc(cspn3d_fwd_f32(fptr(g), fptr(f), out.data_ptr<float>(), B, C, D, H, W, (int)prop_time, (int)norm_type,
                            ws_bytes ? ws.data_ptr() : nullptr, ws_bytes, (cspn_stream_t)c10::cuda::getCurrentCUDAStream().stream()),
             "cspn3d_fwd_f32");
    return out;
}

std::tuple<at::Tensor, at::Tensor> propagate3d_backward_cuda(const at::Tensor& guidance, const at::Tensor& feat,
                                                             const at::Tensor& grad_out, int64_t prop_time, int64_t norm_type,
                                                             bool need_g, bool need_f) {
    check3d(guidance, feat);
    TORCH_CHECK(grad_out.sizes() == feat.sizes() && grad_out.scalar_type() == at::kFloat && grad_out.device() == feat.device(),
                "grad_out must match feat");
    const c10::cuda::CUDAGuard guard(feat.device());
    const at::Tensor g = guidance.contiguous(), f = feat.contiguous(), go = grad_out.contiguous();
    at::Tensor gg = need_g ? at::empty_like(g) : at::Tensor();
    at::Tensor gf = need_f ? at::empty_like(f) : at::Tensor();
    if (prop_time == 0) {
        if (need_g) gg.zero_();
        if (need_f) gf.copy_(go);
        return {need_g ? gg : at::zeros({0}, g.options()), need_f ? gf : at::zeros({0}, f.options())};
    }
    const int B = (int)f.size(0), C = (int)f.size(1), D = (int)f.size(2), H = (int)f.size(3), W = (int)f.size(4);
    const size_t ws_bytes = cspn3d_bwd_workspace_bytes(B, C, D, H, W, (int)prop_time);
    at::Tensor ws;
    if (ws_bytes) ws = at::empty({(int64_t)ws_bytes}, f.options().dtype(at::kByte));
    check_rc(cspn3d_bwd_f32(fptr(g), fptr(f), fptr(go), need_g ? gg.data_ptr<float>() : nullptr, need_f ? gf.data_ptr<float>() : nullptr,
                            B, C, D, H, W, (int)prop_time, (int)norm_type, ws_bytes ? ws.data_ptr() : nullptr, ws_bytes,
                            (cspn_stream_t)c10::cuda::getCurrentCUDAStream().stream()),
             "cspn3d_bwd_f32");
    return {need_g ? gg : at::zeros({0}, g.options()), need_f ? gf : at::zeros({0}, f.options())};
}

// K x K x K kernels: K = 3 is the 3D operator above (same kernels, same bits); K = 5 goes through cspn3d_k_*_f32
void check3d_k(const at::Tensor& guidance, const at::Tensor& feat, int64_t K) {
    TORCH_CHECK_VALUE(K == 3 || K == 5, "3D kernel_size must be 3 or 5, got ", K);
    TORCH_CHECK_VALUE(guidance.dim() == 5 && feat.dim() == 5, "guidance and feat must be (B,C,D,H,W)");
    TORCH_CHECK(guidance.scalar_type() == at::kFloat && feat.scalar_type() == at::kFloat, "cspn_b200 is fp32 only");
    const int64_t nt = K * K * K - 1;
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
    const size_t ws_bytes = cspn3d_k_workspace_bytes(B, C, D, H, W, (int)K, (int)prop_time);
    at::Tensor ws;
    if (ws_bytes) ws = at::empty({(int64_t)ws_bytes}, f.options().dtype(at::kByte));
    check_rc(cspn3d_k_fwd_f32(fptr(g), fptr(f), out.data_ptr<float>(), B, C, D, H, W, (int)K, (int)prop_time, (int)norm_type,
                              ws_bytes ? ws.data_ptr() : nullptr, ws_bytes, (cspn_stream_t)c10::cuda::getCurrentCUDAStream().stream()),
             "cspn3d_k_fwd_f32");
    return out;
}

std::tuple<at::Tensor, at::Tensor> propagate3d_k_backward_cuda(const at::Tensor& guidance, const at::Tensor& feat,
                                                               const at::Tensor& grad_out, int64_t K, int64_t prop_time,
                                                               int64_t norm_type, bool need_g, bool need_f) {
    check3d_k(guidance, feat, K);
    if (K == 3) return propagate3d_backward_cuda(guidance, feat, grad_out, prop_time, norm_type, need_g, need_f);
    TORCH_CHECK(grad_out.sizes() == feat.sizes() && grad_out.scalar_type() == at::kFloat && grad_out.device() == feat.device(),
                "grad_out must match feat");
    const c10::cuda::CUDAGuard guard(feat.device());
    const at::Tensor g = guidance.contiguous(), f = feat.contiguous(), go = grad_out.contiguous();
    at::Tensor gg = need_g ? at::empty_like(g) : at::Tensor();
    at::Tensor gf = need_f ? at::empty_like(f) : at::Tensor();
    const int B = (int)f.size(0), C = (int)f.size(1), D = (int)f.size(2), H = (int)f.size(3), W = (int)f.size(4);
    const size_t ws_bytes = cspn3d_k_bwd_workspace_bytes(B, C, D, H, W, (int)K, (int)prop_time);
    at::Tensor ws;
    if (ws_bytes) ws = at::empty({(int64_t)ws_bytes}, f.options().dtype(at::kByte));
    check_rc(cspn3d_k_bwd_f32(fptr(g), fptr(f), fptr(go), need_g ? gg.data_ptr<float>() : nullptr,
                              need_f ? gf.data_ptr<float>() : nullptr, B, C, D, H, W, (int)K, (int)prop_time, (int)norm_type,
                              ws_bytes ? ws.data_ptr() : nullptr, ws_bytes, (cspn_stream_t)c10::cuda::getCurrentCUDAStream().stream()),
             "cspn3d_k_bwd_f32");
    return {need_g ? gg : at::zeros({0}, g.options()), need_f ? gf : at::zeros({0}, f.options())};
}

// caller-supplied gates (fluid.layers.affinity_propagate), nd = 2 (K in {3, 5, 7}) or 3 (K in {3, 5}).  Returns the
// (images, channels) the C ABI is called with: per-channel gates are B*C images of one channel.
std::pair<int, int> check_gates(const at::Tensor& input, const at::Tensor& gate, int64_t K, int64_t prop_step, int nd) {
    TORCH_CHECK_VALUE(input.dim() == nd + 2 && gate.dim() == nd + 2, "input and gate_weight must be ",
                      nd == 2 ? "(B,C,H,W)" : "(B,C,D,H,W)");
    TORCH_CHECK_VALUE(nd == 2 ? (K == 3 || K == 5 || K == 7) : (K == 3 || K == 5), "kernel_size of a ", nd,
                      "D affinity_propagate must be ", nd == 2 ? "3, 5 or 7" : "3 or 5", ", got ", K);
    TORCH_CHECK_VALUE(prop_step >= 0, "prop_step must be >= 0, got ", prop_step);
    TORCH_CHECK(input.scalar_type() == at::kFloat && gate.scalar_type() == at::kFloat, "cspn_b200 is fp32 only");
    const int64_t nt = (nd == 2 ? K * K : K * K * K) - 1, B = input.size(0), C = input.size(1);
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
    const auto stream = (cspn_stream_t)c10::cuda::getCurrentCUDAStream().stream();
    const int H = (int)x.size(nd), W = (int)x.size(nd + 1), D = nd == 3 ? (int)x.size(2) : 1;
    const size_t ws_bytes = nd == 2 ? cspn2d_gates_workspace_bytes(B, C, H, W, (int)K, (int)prop_step)
                                    : cspn3d_gates_workspace_bytes(B, C, D, H, W, (int)K, (int)prop_step);
    at::Tensor ws;
    if (ws_bytes) ws = at::empty({(int64_t)ws_bytes}, x.options().dtype(at::kByte));
    void* w = ws_bytes ? ws.data_ptr() : nullptr;
    if (nd == 2)
        check_rc(cspn2d_gates_fwd_f32(fptr(g), fptr(x), out.data_ptr<float>(), B, C, H, W, (int)K, (int)prop_step, w, ws_bytes, stream),
                 "cspn2d_gates_fwd_f32");
    else
        check_rc(cspn3d_gates_fwd_f32(fptr(g), fptr(x), out.data_ptr<float>(), B, C, D, H, W, (int)K, (int)prop_step, w, ws_bytes,
                                      stream),
                 "cspn3d_gates_fwd_f32");
    return out;
}

std::tuple<at::Tensor, at::Tensor> affinity_propagate_backward_cuda(const at::Tensor& input, const at::Tensor& gate,
                                                                    const at::Tensor& grad_out, int64_t K, int64_t prop_step,
                                                                    bool need_x, bool need_g, int nd) {
    const auto [B, C] = check_gates(input, gate, K, prop_step, nd);
    TORCH_CHECK(grad_out.sizes() == input.sizes() && grad_out.scalar_type() == at::kFloat && grad_out.device() == input.device(),
                "grad_out must match input");
    const c10::cuda::CUDAGuard guard(input.device());
    const at::Tensor g = gate.contiguous(), x = input.contiguous(), go = grad_out.contiguous();
    at::Tensor gx = need_x ? at::empty_like(x) : at::Tensor();
    at::Tensor gg = need_g ? at::empty_like(g) : at::Tensor();
    const auto stream = (cspn_stream_t)c10::cuda::getCurrentCUDAStream().stream();
    const int H = (int)x.size(nd), W = (int)x.size(nd + 1), D = nd == 3 ? (int)x.size(2) : 1;
    const size_t ws_bytes = nd == 2 ? cspn2d_gates_bwd_workspace_bytes(B, C, H, W, (int)K, (int)prop_step)
                                    : cspn3d_gates_bwd_workspace_bytes(B, C, D, H, W, (int)K, (int)prop_step);
    at::Tensor ws;
    if (ws_bytes) ws = at::empty({(int64_t)ws_bytes}, x.options().dtype(at::kByte));
    void* w = ws_bytes ? ws.data_ptr() : nullptr;
    float* pgg = need_g ? gg.data_ptr<float>() : nullptr;
    float* pgx = need_x ? gx.data_ptr<float>() : nullptr;
    if (nd == 2)
        check_rc(cspn2d_gates_bwd_f32(fptr(g), fptr(x), fptr(go), pgg, pgx, B, C, H, W, (int)K, (int)prop_step, w, ws_bytes, stream),
                 "cspn2d_gates_bwd_f32");
    else
        check_rc(cspn3d_gates_bwd_f32(fptr(g), fptr(x), fptr(go), pgg, pgx, B, C, D, H, W, (int)K, (int)prop_step, w, ws_bytes,
                                      stream),
                 "cspn3d_gates_bwd_f32");
    return {need_x ? gx : at::zeros({0}, x.options()), need_g ? gg : at::zeros({0}, g.options())};
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
    check_rc(cspn_unpool_conv3x3_fwd_f32(fptr(xc), fptr(wc), out.data_ptr<float>(), (int)xc.size(0), (int)xc.size(1), (int)xc.size(2),
                                         (int)xc.size(3), (int)wc.size(0), (int)H, (int)W,
                                         (cspn_stream_t)c10::cuda::getCurrentCUDAStream().stream()),
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
    at::Tensor gx = need_x ? at::empty_like(xc) : at::Tensor();
    at::Tensor gw = need_w ? at::empty_like(wc) : at::Tensor();
    const int B = (int)xc.size(0), Cin = (int)xc.size(1), h = (int)xc.size(2), w = (int)xc.size(3), Cout = (int)wc.size(0);
    const size_t ws_bytes = need_w ? cspn_unpool_conv3x3_bwd_workspace_bytes(B, Cin, h, w, Cout, (int)H, (int)W) : 0;
    at::Tensor ws;
    if (ws_bytes) ws = at::empty({(int64_t)ws_bytes}, xc.options().dtype(at::kByte));
    if (need_x || need_w)
        check_rc(cspn_unpool_conv3x3_bwd_f32(fptr(xc), fptr(wc), fptr(go), need_x ? gx.data_ptr<float>() : nullptr,
                                             need_w ? gw.data_ptr<float>() : nullptr, B, Cin, h, w, Cout, (int)H, (int)W,
                                             ws_bytes ? ws.data_ptr() : nullptr, ws_bytes,
                                             (cspn_stream_t)c10::cuda::getCurrentCUDAStream().stream()),
                 "cspn_unpool_conv3x3_bwd_f32");
    return {need_x ? gx : at::zeros({0}, xc.options()), need_w ? gw : at::zeros({0}, wc.options())};
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
}

TORCH_LIBRARY_IMPL(cspn_b200, CUDA, m) {
    m.impl("propagate2d", &propagate2d_cuda);
    m.impl("propagate2d_backward", &propagate2d_backward_cuda);
    m.impl("propagate2d_k", &propagate2d_k_cuda);
    m.impl("propagate2d_k_backward", &propagate2d_k_backward_cuda);
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
}
