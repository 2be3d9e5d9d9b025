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
//   propagate3d(Tensor guidance, Tensor feat, int prop_time, int norm_type) -> Tensor
//   propagate3d_backward(Tensor guidance, Tensor feat, Tensor grad_out, int prop_time, int norm_type,
//                        bool need_guidance, bool need_feat) -> (Tensor, Tensor)
// There is no CPU kernel: CPU tensors reach the dispatcher's "no kernel for backend CPU" error, loudly.
#include <ATen/ATen.h>
#include <c10/cuda/CUDAGuard.h>
#include <c10/cuda/CUDAStream.h>
#include <torch/library.h>

#include <optional>
#include <tuple>

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

}  // namespace

TORCH_LIBRARY(cspn_b200, m) {
    m.def("propagate2d(Tensor guidance, Tensor blur_depth, Tensor? sparse_depth, int prop_time, int norm_type, int algo) -> Tensor");
    m.def("propagate2d_backward(Tensor guidance, Tensor blur_depth, Tensor? sparse_depth, Tensor grad_out, int prop_time, "
          "int norm_type, bool need_guidance, bool need_blur) -> (Tensor, Tensor)");
    m.def("propagate3d(Tensor guidance, Tensor feat, int prop_time, int norm_type) -> Tensor");
    m.def("propagate3d_backward(Tensor guidance, Tensor feat, Tensor grad_out, int prop_time, int norm_type, "
          "bool need_guidance, bool need_feat) -> (Tensor, Tensor)");
}

TORCH_LIBRARY_IMPL(cspn_b200, CUDA, m) {
    m.impl("propagate2d", &propagate2d_cuda);
    m.impl("propagate2d_backward", &propagate2d_backward_cuda);
    m.impl("propagate3d", &propagate3d_cuda);
    m.impl("propagate3d_backward", &propagate3d_backward_cuda);
}
