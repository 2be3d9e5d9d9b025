// Dynamic K x K propagation with per-step attention over the distance rings and an anchor to the initial depth: DySPN's
// step (Lin et al., AAAI 2022; DESIGN.md section 4.23).  affinity (B, K*K, H, W) holds all K*K taps, the centre included,
// as given, shared by the C channels; channel j = i*K + l weights d_t(p + o_j), o_j = (i - R, l - R), R = (K - 1) / 2
// (F.unfold's row order).  Tap j lies on ring(j) = max(|i - R|, |l - R|): ring 0 is the centre, ring r holds 8r taps.
// attention (B, N*(R+1), H, W) holds, in channel t*(R+1) + r, the attention of ring r at step t, as given.  blur
// (B, C, H, W) is d_0; sparse s and confidence m are (B, 1, H, W), both or neither.  A read outside the image is 0.
//
//   w_{t,j}(p) = a_{t,ring(j)}(p) * affinity_j(p)                        (one rounded product, recomputed where needed)
//   rho_t(p)   = 1 - S,  S = w_0 + w_1 + ... + w_{K*K-1}                  (adds, j ascending)
//   v_t(p)     = fma over j = K*K-1 down to 0 of w_{t,j}(p) * d_t(p + o_j), starting from rho_t(p) * d_0(p)
//   d_{t+1}(p) = m*s + (1 - m)*v_t(p)       (with samples; d_{t+1} = v_t without), out = d_N
//
// Every product outside the FMA chain and every sum is rounded on its own.  The tap order is the dilated step's (section
// 4.22): with attention 1 and a zero centre affinity a step gives propagate2d_dilated's bits at dilation 1 when that op's
// centre weight is rho.  Neither the attention nor the confidence is folded into a precombined weight, so the NaN and
// +-inf masks are the composition's.
//
// Backward, lambda_N = grad_out, mu_t = (1 - m) * lambda_{t+1} (lambda_{t+1} without samples):
//   lambda_t(q)   = fma over j = K*K-1 down to 0, source q - o_j inside the image, of w_{t,j} * mu_t there
//   grad_blur     = lambda_0 + sum_t rho_t mu_t                                           (fma, t ascending)
//   g_{t,j}(p)    = G1 - G0,  G1 = sum_c mu_t d_t(p + o_j),  G0 = sum_c mu_t d_0            (fma, c ascending; a tap
//                   outside the image adds mu * 0)
//   grad_affinity_j    = sum_t a_{t,ring(j)} g_{t,j}                                      (fma, t ascending)
//   grad_attention_t,r = sum_{j in ring r} affinity_j g_{t,j}                             (fma, j ascending)
//   grad_conf(p)  = sum_t ((sum_c lambda_{t+1}) s - sum_c lambda_{t+1} v_t),  grad_sparse(p) = sum_t m sum_c lambda_{t+1}
//                   (t then c ascending; the lambda sum by adds, the lambda v sum by fma), v_t recomputed in the
//                   forward's order
// Only an affinity, attention or confidence gradient needs d_1 .. d_{N-1}.
//
// Kernels (sm_90a), on the dilated step's tiles and helpers (cspn2d_stencil.cuh):
//   step      one launch per step, grid z = image * channel; a tile of d_t with an R halo staged in shared memory; 4 pixels
//             per thread with LDG.128 planes when W % 4 == 0 and the planes are 16-byte aligned, else 1; both give the
//             same bits.  The affinity is read twice per pixel, once for S and once for the taps; the second read is
//             meant to hit the cache.
//   adjoint   one launch per step, the transposed stencil over a staged tile of mu_t, one pixel per thread;
//   finalize  one launch: a slice per kernel row for grad_affinity, up to kAttSlices slices over the steps for
//             grad_attention, and one slice for the per-pixel rest, each thread over all channels (and steps).
//             Each slice recomputes the g it needs from the stored iterates, so every accumulator stays in registers.
// No atomics and no memsets (except the N = 0 backward's zero gradients); every output word is written by one thread.
#include "cspn2d_stencil.cuh"

namespace cspn {
namespace {

constexpr int kTX = 32, kTY = 8, kRows = 2;          // the dilated step's tile: threads per CTA (x, y), rows per thread
constexpr int kTH = kTY * kRows;                     // tile height
constexpr int kFinThreads = 128;
constexpr int kAttSlices = 64;                       // grid slices of grad_attention; slice z takes steps z, z + 64, ...

// a[r] for a run-time r < NR, by selects: the array stays in registers
template <int NR, typename T>
__device__ __forceinline__ T pick(const T (&a)[NR], int r) {
    T v = a[0];
#pragma unroll
    for (int q = 1; q < NR; ++q)
        if (r == q) v = a[q];
    return v;
}

template <int K>
__host__ __device__ constexpr int ring_of(int j) {
    const int R = (K - 1) / 2, di = j / K - R, dl = j % K - R;
    const int ai = di < 0 ? -di : di, al = dl < 0 ? -dl : dl;
    return ai > al ? ai : al;
}

// d_{t+1} from d_t (cur, staged), d_0, the affinity and step t's R + 1 attention planes (att: image 0's ring 0 of step t;
// image b's at att + b * att_ch * HW)
template <int K, int VEC, bool SAMP>
__global__ void __launch_bounds__(kTX * kTY)
dyn_step_kernel(const float* __restrict__ aff, const float* __restrict__ att, const float* __restrict__ d0,
                const float* __restrict__ cur, const float* __restrict__ sparse, const float* __restrict__ conf, float* __restrict__ dst,
                int C, int H, int W, int att_ch) {
    constexpr int R = (K - 1) / 2, KK = K * K, NR = R + 1;
    extern __shared__ float tile[];
    const int TW = kTX * VEC, pitch = TW + 2 * R;
    const int x0 = blockIdx.x * TW, y0 = blockIdx.y * kTH, bc = blockIdx.z, b = bc / C;
    const size_t HW = (size_t)H * W;
    stage<kTX, kTY, kTH>(tile, pitch, cur + (size_t)bc * HW, nullptr, x0, y0, R, H, W);
    __syncthreads();
    const float* wk = aff + (size_t)b * KK * HW;
    const float* wa = att + (size_t)b * att_ch * HW;
    const int tx = threadIdx.x * VEC, x = x0 + tx;
    if (x >= W) return;
#pragma unroll 1
    for (int r = 0; r < kRows; ++r) {
        const int ty = threadIdx.y + r * kTY, y = y0 + ty;
        if (y >= H) return;
        const size_t p = (size_t)y * W + x, o = (size_t)bc * HW + p;
        const float* t0 = tile + (ty + R) * pitch + tx + R;
        if constexpr (VEC == 4) {
            float4 a[NR];
#pragma unroll
            for (int q = 0; q < NR; ++q) a[q] = ld4(wa + q * HW + p);
            // one kernel row per iteration: unrolled over all K*K taps, the compiler would hoist every load (254 registers)
            float4 S = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll 1
            for (int i = 0; i < K; ++i) {
                const int ai = i < R ? R - i : i - R;
#pragma unroll
                for (int l = 0; l < K; ++l) {
                    const int al = l < R ? R - l : l - R;
                    const float4 f = ld4(wk + (i * K + l) * HW + p), ar = pick(a, ai > al ? ai : al);
                    const float4 w = make_float4(__fmul_rn(ar.x, f.x), __fmul_rn(ar.y, f.y), __fmul_rn(ar.z, f.z), __fmul_rn(ar.w, f.w));
                    const bool first = i == 0 && l == 0;
                    S = make_float4(first ? w.x : __fadd_rn(S.x, w.x), first ? w.y : __fadd_rn(S.y, w.y),
                                    first ? w.z : __fadd_rn(S.z, w.z), first ? w.w : __fadd_rn(S.w, w.w));
                }
            }
            const float4 dd = ld4(d0 + o);
            float v0 = __fmul_rn(__fsub_rn(1.f, S.x), dd.x), v1 = __fmul_rn(__fsub_rn(1.f, S.y), dd.y);
            float v2 = __fmul_rn(__fsub_rn(1.f, S.z), dd.z), v3 = __fmul_rn(__fsub_rn(1.f, S.w), dd.w);
#pragma unroll 1
            for (int i = K - 1; i >= 0; --i) {                        // j = i*K + l descending
                const int ai = i < R ? R - i : i - R;
#pragma unroll
                for (int l = K - 1; l >= 0; --l) {
                    const int al = l < R ? R - l : l - R;
                    const float4 f = ld4(wk + (i * K + l) * HW + p), ar = pick(a, ai > al ? ai : al);
                    const float* s = t0 + (i - R) * pitch + (l - R);
                    v0 = fmaf(__fmul_rn(ar.x, f.x), s[0], v0);
                    v1 = fmaf(__fmul_rn(ar.y, f.y), s[1], v1);
                    v2 = fmaf(__fmul_rn(ar.z, f.z), s[2], v2);
                    v3 = fmaf(__fmul_rn(ar.w, f.w), s[3], v3);
                }
            }
            if constexpr (SAMP) {
                const float4 m = ld4(conf + (size_t)b * HW + p), sv = ld4(sparse + (size_t)b * HW + p);
                v0 = blend(m.x, sv.x, v0);
                v1 = blend(m.y, sv.y, v1);
                v2 = blend(m.z, sv.z, v2);
                v3 = blend(m.w, sv.w, v3);
            }
            *reinterpret_cast<float4*>(dst + o) = make_float4(v0, v1, v2, v3);
        } else {
            float a[NR];
#pragma unroll
            for (int q = 0; q < NR; ++q) a[q] = __ldg(wa + q * HW + p);
            float S = 0.f;
#pragma unroll
            for (int j = 0; j < KK; ++j) {
                const float w = __fmul_rn(a[ring_of<K>(j)], __ldg(wk + j * HW + p));
                S = j == 0 ? w : __fadd_rn(S, w);
            }
            float v = __fmul_rn(__fsub_rn(1.f, S), __ldg(d0 + o));
#pragma unroll
            for (int j = KK - 1; j >= 0; --j)
                v = fmaf(__fmul_rn(a[ring_of<K>(j)], __ldg(wk + j * HW + p)), t0[(j / K - R) * pitch + (j % K - R)], v);
            if constexpr (SAMP) v = blend(__ldg(conf + (size_t)b * HW + p), __ldg(sparse + (size_t)b * HW + p), v);
            dst[o] = v;
        }
    }
}

// lambda_t(q) = sum_j w_{t,j}(q - o_j) mu_t(q - o_j), sources inside the image only; mu_t = (1 - m) lambda_{t+1} (conf) or
// lambda_{t+1}
template <int K>
__global__ void __launch_bounds__(kTX * kTY)
dyn_adjoint_kernel(const float* __restrict__ aff, const float* __restrict__ att, const float* __restrict__ lam_in,
                   const float* __restrict__ conf, float* __restrict__ lam_out, int C, int H, int W, int att_ch) {
    constexpr int R = (K - 1) / 2, KK = K * K;
    extern __shared__ float tile[];
    const int pitch = kTX + 2 * R;
    const int x0 = blockIdx.x * kTX, y0 = blockIdx.y * kTH, bc = blockIdx.z, b = bc / C;
    const size_t HW = (size_t)H * W;
    stage<kTX, kTY, kTH>(tile, pitch, lam_in + (size_t)bc * HW, conf ? conf + (size_t)b * HW : nullptr, x0, y0, R, H, W);
    __syncthreads();
    const float* wk = aff + (size_t)b * KK * HW;
    const float* wa = att + (size_t)b * att_ch * HW;
    const int tx = threadIdx.x, x = x0 + tx;
    if (x >= W) return;
#pragma unroll 1
    for (int r = 0; r < kRows; ++r) {
        const int ty = threadIdx.y + r * kTY, y = y0 + ty;
        if (y >= H) return;
        const float* t0 = tile + (ty + R) * pitch + tx + R;
        float acc = 0.f;
#pragma unroll 1
        for (int i = K - 1; i >= 0; --i) {                            // j = i*K + l descending
            const int oy = i - R, ys = y - oy, ai = oy < 0 ? -oy : oy;
#pragma unroll
            for (int l = K - 1; l >= 0; --l) {
                const int ox = l - R, xs = x - ox, al = ox < 0 ? -ox : ox;
                if (in_image(ys, xs, H, W)) {
                    const size_t q = (size_t)ys * W + xs;
                    const float w = __fmul_rn(__ldg(wa + (ai > al ? ai : al) * HW + q), __ldg(wk + (i * K + l) * HW + q));
                    acc = fmaf(w, t0[-oy * pitch - ox], acc);
                }
            }
        }
        lam_out[(size_t)bc * HW + (size_t)y * W + x] = acc;
    }
}

// The gradients of pixel p of image b.  lams holds lambda_0 .. lambda_{N-1} (lambda_N is grad_out), iters d_1 .. d_{N-1}
// (d_0 is blur), each P = B*C*H*W floats.  Grid z: z_aff slices (K when grad_aff is wanted, else 0), slice i forming
// grad_affinity of kernel row i; then z_att slices (min(N, kAttSlices) when grad_att is wanted, else 0), slice z forming
// grad_attention of steps z, z + z_att, ...; then one slice for grad_blur, grad_sparse and grad_conf.  Without ITER,
// z_aff = z_att = 0 and no iterate is read.
template <int K, bool SAMP, bool ITER>
__global__ void __launch_bounds__(kFinThreads)
dyn_finalize_kernel(const float* __restrict__ aff, const float* __restrict__ att, const float* __restrict__ d0,
                    const float* __restrict__ sparse, const float* __restrict__ conf, const float* __restrict__ grad_out,
                    const float* __restrict__ iters, const float* __restrict__ lams, float* __restrict__ grad_aff,
                    float* __restrict__ grad_att, float* __restrict__ grad_blur, float* __restrict__ grad_sparse,
                    float* __restrict__ grad_conf, int N, size_t P, int C, int H, int W, int z_aff, int z_att) {
    constexpr int R = (K - 1) / 2, KK = K * K, NR = R + 1;
    const size_t HW = (size_t)H * W;
    const long long pl = (long long)blockIdx.x * kFinThreads + threadIdx.x;
    if (pl >= (long long)HW) return;
    const size_t p = (size_t)pl;
    const int b = blockIdx.y, y = (int)(p / W), x = (int)(p % W), z = blockIdx.z;
    const float* wk = aff + (size_t)b * KK * HW + p;
    const float* wa = att + (size_t)b * N * NR * HW + p;            // step t, ring r at wa[(t*NR + r) * HW]
    const float m = SAMP ? __ldg(conf + (size_t)b * HW + p) : 0.f;
    const float a = SAMP ? __fsub_rn(1.f, m) : 1.f;
    auto lam = [&](int t, size_t o) { return t == N ? __ldg(grad_out + o) : __ldg(lams + (size_t)t * P + o); };
    auto mu = [&](int t, size_t o) { const float l = lam(t + 1, o); return SAMP ? __fmul_rn(a, l) : l; };
    auto iterate = [&](int t, size_t plane) { return t == 0 ? d0 + plane : iters + (size_t)(t - 1) * P + plane; };
    auto weight = [&](int t, int j) { return __fmul_rn(__ldg(wa + ((size_t)t * NR + ring_of<K>(j)) * HW), __ldg(wk + j * HW)); };
    auto rho = [&](int t) {
        float S = weight(t, 0);
#pragma unroll
        for (int j = 1; j < KK; ++j) S = __fadd_rn(S, weight(t, j));
        return __fsub_rn(1.f, S);
    };
    auto g0 = [&](int t) {                                          // sum_c mu_t d_0(p)
        float g = 0.f;
        for (int c = 0; c < C; ++c) {
            const size_t plane = ((size_t)b * C + c) * HW;
            g = fmaf(mu(t, plane + p), __ldg(d0 + plane + p), g);
        }
        return g;
    };
    auto g1 = [&](int t, int j) {                                   // sum_c mu_t d_t(p + o_j)
        const int ys = y + j / K - R, xs = x + j % K - R;
        const bool inside = in_image(ys, xs, H, W);
        float g = 0.f;
        for (int c = 0; c < C; ++c) {
            const size_t plane = ((size_t)b * C + c) * HW;
            g = fmaf(mu(t, plane + p), inside ? __ldg(iterate(t, plane) + (size_t)ys * W + xs) : 0.f, g);
        }
        return g;
    };
    if (ITER && z < z_aff) {
        const int i = z;
        float ga[K];
#pragma unroll
        for (int l = 0; l < K; ++l) ga[l] = 0.f;
        for (int t = 0; t < N; ++t) {
            const float G0 = g0(t);
#pragma unroll
            for (int l = 0; l < K; ++l) {
                const int j = i * K + l;
                ga[l] = fmaf(__ldg(wa + ((size_t)t * NR + ring_of<K>(j)) * HW), __fsub_rn(g1(t, j), G0), ga[l]);
            }
        }
#pragma unroll
        for (int l = 0; l < K; ++l) grad_aff[((size_t)b * KK + i * K + l) * HW + p] = ga[l];
        return;
    }
    if (ITER && z < z_aff + z_att) {
        for (int t = z - z_aff; t < N; t += z_att) {
            const float G0 = g0(t);
            float gr[NR];
#pragma unroll
            for (int q = 0; q < NR; ++q) gr[q] = 0.f;
#pragma unroll
            for (int j = 0; j < KK; ++j) gr[ring_of<K>(j)] = fmaf(__ldg(wk + j * HW), __fsub_rn(g1(t, j), G0), gr[ring_of<K>(j)]);
#pragma unroll
            for (int q = 0; q < NR; ++q) grad_att[((size_t)b * N * NR + (size_t)t * NR + q) * HW + p] = gr[q];
        }
        return;
    }
    if (grad_blur) {
        for (int c = 0; c < C; ++c) {
            const size_t o = ((size_t)b * C + c) * HW + p;
            float g = __ldg(lams + o);
            for (int t = 0; t < N; ++t) g = fmaf(rho(t), mu(t, o), g);
            grad_blur[o] = g;
        }
    }
    if constexpr (SAMP) {
        if (!grad_sparse && !grad_conf) return;
        const float s = __ldg(sparse + (size_t)b * HW + p);
        float gm = 0.f, gs = 0.f;
        for (int t = 0; t < N; ++t) {
            const float rt = (ITER && grad_conf) ? rho(t) : 0.f;
            float A = 0.f, Bs = 0.f;
            for (int c = 0; c < C; ++c) {
                const size_t plane = ((size_t)b * C + c) * HW;
                const float l0 = lam(t + 1, plane + p);
                A = __fadd_rn(A, l0);
                if (ITER && grad_conf) {
                    const float* dt = iterate(t, plane);
                    float v = __fmul_rn(rt, __ldg(d0 + plane + p));
#pragma unroll 1
                    for (int i = K - 1; i >= 0; --i) {                // j = i*K + l descending, the forward's order
                        const int ys = y + i - R;
#pragma unroll
                        for (int l = K - 1; l >= 0; --l) {
                            const int xs = x + l - R;
                            v = fmaf(weight(t, i * K + l), in_image(ys, xs, H, W) ? __ldg(dt + (size_t)ys * W + xs) : 0.f, v);
                        }
                    }
                    Bs = fmaf(l0, v, Bs);
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
int launch_step(bool vec, const float* aff, const float* att_t, const float* d0, const float* cur, const float* sparse, const float* conf,
                float* dst, int B, int C, int H, int W, int att_ch, cudaStream_t st) {
    const int VEC = vec ? 4 : 1;
    const dim3 grid((unsigned)ceil_div(W, kTX * VEC), (unsigned)ceil_div(H, kTH), (unsigned)(B * C)), block(kTX, kTY);
    const size_t sm = tile_smem(VEC, (K - 1) / 2);
    if (vec && sparse)
        dyn_step_kernel<K, 4, true><<<grid, block, sm, st>>>(aff, att_t, d0, cur, sparse, conf, dst, C, H, W, att_ch);
    else if (vec)
        dyn_step_kernel<K, 4, false><<<grid, block, sm, st>>>(aff, att_t, d0, cur, sparse, conf, dst, C, H, W, att_ch);
    else if (sparse)
        dyn_step_kernel<K, 1, true><<<grid, block, sm, st>>>(aff, att_t, d0, cur, sparse, conf, dst, C, H, W, att_ch);
    else
        dyn_step_kernel<K, 1, false><<<grid, block, sm, st>>>(aff, att_t, d0, cur, sparse, conf, dst, C, H, W, att_ch);
    CSPN_CUDA_TRY(cudaGetLastError());
    return CSPN_OK;
}

template <int K>
int forward_k(const float* aff, const float* att, const float* blur, const float* sparse, const float* conf, float* out, int B, int C,
              int H, int W, int N, void* ws, cudaStream_t st, int* launches) {
    constexpr int NR = (K + 1) / 2;
    const size_t HW = (size_t)H * W;
    float* buf = static_cast<float*>(ws);
    const bool vec = vec_ok(W, {aff, att, blur, sparse, conf, out, N > 1 ? buf : nullptr});
    const float* cur = blur;
    for (int t = 0; t < N; ++t) {
        float* dst = ((N - 1 - t) & 1) ? buf : out;      // d_N lands in out; the others alternate with the one buffer
        const int rc = launch_step<K>(vec, aff, att + (size_t)t * NR * HW, blur, cur, sparse, conf, dst, B, C, H, W, N * NR, st);
        if (rc != CSPN_OK) return rc;
        cur = dst;
    }
    *launches = N;
    return CSPN_OK;
}

template <int K>
int backward_k(const float* aff, const float* att, const float* blur, const float* sparse, const float* conf, const float* grad_out,
               float* grad_aff, float* grad_att, float* grad_blur, float* grad_sparse, float* grad_conf, int B, int C, int H, int W, int N,
               void* ws, cudaStream_t st, int* launches) {
    constexpr int NR = (K + 1) / 2;
    const size_t HW = (size_t)H * W, P = (size_t)B * C * HW;
    float* lams = static_cast<float*>(ws);                   // lambda_0 .. lambda_{N-1}
    float* iters = lams + (size_t)N * P;                     // d_1 .. d_{N-1}
    const bool iter = grad_aff || grad_att || grad_conf;
    int nl = 0;
    if (iter) {
        const bool vec = vec_ok(W, {aff, att, blur, sparse, conf, N > 1 ? iters : nullptr});
        for (int t = 0; t + 1 < N; ++t) {
            const int rc = launch_step<K>(vec, aff, att + (size_t)t * NR * HW, blur, t == 0 ? blur : iters + (size_t)(t - 1) * P, sparse,
                                          conf, iters + (size_t)t * P, B, C, H, W, N * NR, st);
            if (rc != CSPN_OK) return rc;
            ++nl;
        }
    }
    const int t_end = grad_blur ? 0 : 1;                      // lambda_0 feeds grad_blur only
    const dim3 grid((unsigned)ceil_div(W, kTX), (unsigned)ceil_div(H, kTH), (unsigned)(B * C)), block(kTX, kTY);
    for (int t = N - 1; t >= t_end; --t) {
        dyn_adjoint_kernel<K><<<grid, block, tile_smem(1, (K - 1) / 2), st>>>(aff, att + (size_t)t * NR * HW,
                                                                 t + 1 == N ? grad_out : lams + (size_t)(t + 1) * P, conf,
                                                                 lams + (size_t)t * P, C, H, W, N * NR);
        CSPN_CUDA_TRY(cudaGetLastError());
        ++nl;
    }
    const int z_aff = grad_aff ? K : 0, z_att = grad_att ? (N < kAttSlices ? N : kAttSlices) : 0;
    const dim3 fg((unsigned)ceil_div((long long)H * W, kFinThreads), (unsigned)B, (unsigned)(z_aff + z_att + 1));
#define CSPN_DYN_FIN(S, I)                                                                                                        \
    dyn_finalize_kernel<K, S, I><<<fg, kFinThreads, 0, st>>>(aff, att, blur, sparse, conf, grad_out, iters, lams, grad_aff, grad_att, \
                                                             grad_blur, grad_sparse, grad_conf, N, P, C, H, W, z_aff, z_att)
    if (sparse && iter) CSPN_DYN_FIN(true, true);
    else if (sparse) CSPN_DYN_FIN(true, false);
    else if (iter) CSPN_DYN_FIN(false, true);
    else CSPN_DYN_FIN(false, false);
#undef CSPN_DYN_FIN
    CSPN_CUDA_TRY(cudaGetLastError());
    *launches = nl + 1;
    return CSPN_OK;
}

}  // namespace

int dynamic2d_launchable(int B, int C, int H, int W, const char** why) {
    if ((long long)B * C > 65535) { *why = "B*C exceeds gridDim.z (65535)"; return 0; }
    if (ceil_div(H, kTH) > 65535) { *why = "ceil(H/16) exceeds gridDim.y (65535)"; return 0; }
    return 1;
}

size_t dynamic2d_workspace_bytes(int B, int C, int H, int W, int N) {
    return N >= 2 ? (size_t)B * C * H * W * sizeof(float) : 0;
}

size_t dynamic2d_bwd_workspace_bytes(int B, int C, int H, int W, int N) {
    return N >= 1 ? (size_t)(2 * (size_t)N - 1) * B * C * H * W * sizeof(float) : 0;
}

int dynamic2d_forward(const float* aff, const float* att, const float* blur, const float* sparse, const float* conf, float* out, int B,
                      int C, int H, int W, int K, int N, void* ws, cudaStream_t st, int* launches) {
    if (N == 0) {
        CSPN_CUDA_TRY(cudaMemcpyAsync(out, blur, (size_t)B * C * H * W * sizeof(float), cudaMemcpyDeviceToDevice, st));
        *launches = 0;
        return CSPN_OK;
    }
    switch (K) {
        case 3: return forward_k<3>(aff, att, blur, sparse, conf, out, B, C, H, W, N, ws, st, launches);
        case 5: return forward_k<5>(aff, att, blur, sparse, conf, out, B, C, H, W, N, ws, st, launches);
        default: return forward_k<7>(aff, att, blur, sparse, conf, out, B, C, H, W, N, ws, st, launches);
    }
}

int dynamic2d_backward(const float* aff, const float* att, const float* blur, const float* sparse, const float* conf,
                       const float* grad_out, float* grad_aff, float* grad_att, float* grad_blur, float* grad_sparse, float* grad_conf,
                       int B, int C, int H, int W, int K, int N, void* ws, cudaStream_t st, int* launches) {
    if (N == 0) {      // d_0 = blur: the identity, and nothing reaches the affinity or the samples (zero-filled by memsets);
        const size_t hw = (size_t)H * W;                      // the attention has no channels
        if (grad_blur) CSPN_CUDA_TRY(cudaMemcpyAsync(grad_blur, grad_out, (size_t)B * C * hw * 4, cudaMemcpyDeviceToDevice, st));
        if (grad_aff) CSPN_CUDA_TRY(cudaMemsetAsync(grad_aff, 0, (size_t)B * K * K * hw * 4, st));
        if (grad_sparse) CSPN_CUDA_TRY(cudaMemsetAsync(grad_sparse, 0, (size_t)B * hw * 4, st));
        if (grad_conf) CSPN_CUDA_TRY(cudaMemsetAsync(grad_conf, 0, (size_t)B * hw * 4, st));
        *launches = 0;
        return CSPN_OK;
    }
    switch (K) {
        case 3: return backward_k<3>(aff, att, blur, sparse, conf, grad_out, grad_aff, grad_att, grad_blur, grad_sparse, grad_conf, B, C, H,
                                     W, N, ws, st, launches);
        case 5: return backward_k<5>(aff, att, blur, sparse, conf, grad_out, grad_aff, grad_att, grad_blur, grad_sparse, grad_conf, B, C, H,
                                     W, N, ws, st, launches);
        default: return backward_k<7>(aff, att, blur, sparse, conf, grad_out, grad_aff, grad_att, grad_blur, grad_sparse, grad_conf, B, C,
                                      H, W, N, ws, st, launches);
    }
}

}  // namespace cspn
